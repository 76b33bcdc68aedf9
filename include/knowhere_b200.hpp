// knowhere_b200.hpp — C++ host-side mirror of the reference's operator interface for the hot path,
// header-only over the C ABI (include/knowhere_b200.h).  Same names, argument meaning and error
// behaviour as the reference so that caller code and tests read the same:
//
//   knowhere::Status / expected<T>            include/knowhere/expected.h:34-68,100-200
//   knowhere::Json                            (nlohmann::json in the reference; flat objects only here)
//   knowhere::DataSet, GenDataSet, GenResultDataSet   include/knowhere/dataset.h:452-524
//   knowhere::BitsetView                      include/knowhere/bitsetview.h:131-175
//   knowhere::BinarySet                       include/knowhere/binaryset.h
//   knowhere::IndexNode, Index<IndexNode>     include/knowhere/index/index_node.h:69-395, index/index.h:23-253
//   knowhere::IndexFactory (+ registration)   include/knowhere/index/index_factory.h:27-165
//   knowhere::BruteForce                      include/knowhere/comp/brute_force.h:26-69
//   parameter names (meta::, indexparam::)    include/knowhere/comp/index_param.h:27-78
//
// Every method is noexcept and returns Status / expected<> exactly like the reference facade
// (src/index/index.cc:159-420 wraps node calls in GuardedCall, expected.h:408-430).
#pragma once
#include <algorithm>
#include <cctype>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <string>
#include <utility>
#include <variant>
#include <vector>

#include "knowhere_b200.h"

namespace knowhere {

// ------------------------------------------------------------------ Status / expected
enum class Status {
    success = 0, invalid_args = 1, invalid_param_in_json = 2, out_of_range_in_json = 3, type_conflict_in_json = 4,
    invalid_metric_type = 5, empty_index = 6, not_implemented = 7, index_not_trained = 8, index_already_trained = 9,
    faiss_inner_error = 10, hnsw_inner_error = 12, malloc_error = 13, invalid_binary_set = 19,
    cuda_runtime_error = 22, invalid_index_error = 23, internal_error = 27, emb_list_inner_error = 31,
};

template <typename T>
class expected {
 public:
    expected(const T& v) : val_(v), err_(Status::success) {}
    expected(T&& v) : val_(std::move(v)), err_(Status::success) {}
    static expected<T> Err(Status s, std::string msg) { expected<T> e; e.err_ = s; e.msg_ = std::move(msg); return e; }
    bool has_value() const { return err_ == Status::success; }
    Status error() const { return err_; }
    const T& value() const { return val_; }
    T& value() { return val_; }
    const std::string& what() const { return msg_; }
 private:
    expected() : err_(Status::internal_error) {}
    T val_{};
    Status err_;
    std::string msg_;
};

// ------------------------------------------------------------------ parameter names
namespace meta {
constexpr const char* DIM = "dim";
constexpr const char* ROWS = "rows";
constexpr const char* TOPK = "k";
constexpr const char* METRIC_TYPE = "metric_type";
constexpr const char* RADIUS = "radius";
constexpr const char* RANGE_FILTER = "range_filter";
constexpr const char* EMB_LIST_OFFSET = "EMB_LIST_OFFSET";   // const size_t* [lists + 1] (index_param.h:127)
constexpr const char* EMB_LIST_META = "EMB_LIST_META";       // BinarySet entry of an emb-list index (index_param.h:126)
constexpr const char* EMB_LIST_STRATEGY_TOKENANN = "tokenann";   // index_param.h:131
constexpr const char* EMB_LIST_STRATEGY_MUVERA = "muvera";
constexpr const char* EMB_LIST_STRATEGY = "emb_list_strategy";   // build keys of the strategy (config.h:636-655,836-855):
constexpr const char* EMB_LIST_RERANK = "emb_list_rerank";       // also muvera_num_projections, muvera_num_repeats, muvera_seed
constexpr const char* RETRIEVAL_ANN_RATIO = "retrieval_ann_ratio";
}  // namespace meta
namespace indexparam {
constexpr const char* NLIST = "nlist";
constexpr const char* NPROBE = "nprobe";
constexpr const char* M = "m";
constexpr const char* NBITS = "nbits";
constexpr const char* HNSW_M = "M";
constexpr const char* EFCONSTRUCTION = "efConstruction";
constexpr const char* EF = "ef";
constexpr const char* REFINE = "refine";
constexpr const char* REFINE_K = "refine_k";
constexpr const char* REFINE_TYPE = "refine_type";
}  // namespace indexparam
namespace metric {
constexpr const char* L2 = "L2";
constexpr const char* IP = "IP";
constexpr const char* COSINE = "COSINE";
// emb-list metrics (index_param.h:280-285); MAX_SIM is MAX_SIM_COSINE.  HAMMING / JACCARD need binary vectors, which this
// library does not have: searches with them return invalid_metric_type.
constexpr const char* MAX_SIM = "MAX_SIM";
constexpr const char* MAX_SIM_COSINE = "MAX_SIM_COSINE";
constexpr const char* MAX_SIM_IP = "MAX_SIM_IP";
constexpr const char* MAX_SIM_L2 = "MAX_SIM_L2";
constexpr const char* MAX_SIM_HAMMING = "MAX_SIM_HAMMING";
constexpr const char* MAX_SIM_JACCARD = "MAX_SIM_JACCARD";
}  // namespace metric
namespace IndexEnum {
constexpr const char* INDEX_FAISS_IDMAP = "FLAT";
constexpr const char* INDEX_FAISS_IVFFLAT = "IVF_FLAT";
constexpr const char* INDEX_FAISS_IVFPQ = "IVF_PQ";
constexpr const char* INDEX_HNSW = "HNSW";
}  // namespace IndexEnum

// ------------------------------------------------------------------ Json (flat object)
class Json {
 public:
    using Value = std::variant<std::monostate, bool, int64_t, double, std::string>;
    class Ref {
     public:
        explicit Ref(Value& v) : v_(v) {}
        Ref& operator=(bool b) { v_ = b; return *this; }
        Ref& operator=(int b) { v_ = (int64_t)b; return *this; }
        Ref& operator=(int64_t b) { v_ = b; return *this; }
        Ref& operator=(size_t b) { v_ = (int64_t)b; return *this; }
        Ref& operator=(float b) { v_ = (double)b; return *this; }
        Ref& operator=(double b) { v_ = b; return *this; }
        Ref& operator=(const char* s) { v_ = std::string(s); return *this; }
        Ref& operator=(const std::string& s) { v_ = s; return *this; }
     private:
        Value& v_;
    };
    Ref operator[](const std::string& k) { return Ref(kv_[k]); }
    bool contains(const std::string& k) const { return kv_.count(k) != 0; }
    template <typename T> T get(const std::string& k, T dflt) const {
        auto it = kv_.find(k);
        if (it == kv_.end()) return dflt;
        if (auto p = std::get_if<int64_t>(&it->second)) return (T)*p;
        if (auto p = std::get_if<double>(&it->second)) return (T)*p;
        if (auto p = std::get_if<bool>(&it->second)) return (T)*p;
        return dflt;
    }
    std::string get_string(const std::string& k, const std::string& dflt) const {
        auto it = kv_.find(k);
        if (it == kv_.end()) return dflt;
        if (auto p = std::get_if<std::string>(&it->second)) return *p;
        return dflt;
    }
    std::string dump() const {
        std::ostringstream os;
        os.precision(9);
        os << "{";
        bool first = true;
        for (auto& [k, v] : kv_) {
            if (std::holds_alternative<std::monostate>(v)) continue;
            if (!first) os << ",";
            first = false;
            os << "\"" << k << "\":";
            if (auto p = std::get_if<bool>(&v)) os << (*p ? "true" : "false");
            else if (auto p = std::get_if<int64_t>(&v)) os << *p;
            else if (auto p = std::get_if<double>(&v)) os << *p;
            else if (auto p = std::get_if<std::string>(&v)) os << "\"" << *p << "\"";
        }
        os << "}";
        return os.str();
    }
 private:
    std::map<std::string, Value> kv_;
};

// ------------------------------------------------------------------ DataSet
class DataSet {
 public:
    ~DataSet() {
        if (is_owner_) {
            delete[] ids_; delete[] dist_; delete[] lims_;
            if (owned_tensor_) delete[] (float*)tensor_;
        }
    }
    void SetRows(int64_t r) { rows_ = r; }
    void SetDim(int64_t d) { dim_ = d; }
    void SetTensor(const void* t) { tensor_ = t; }
    void SetIds(const int64_t* p) { ids_ = p; }
    void SetDistance(const float* p) { dist_ = p; }
    void SetLims(const size_t* p) { lims_ = p; }
    void SetIsOwner(bool o) { is_owner_ = o; }
    void SetOwnedTensor(bool o) { owned_tensor_ = o; }
    void SetJsonInfo(std::string j) { json_info_ = std::move(j); }
    const std::string& GetJsonInfo() const { return json_info_; }
    int64_t GetRows() const { return rows_; }
    int64_t GetDim() const { return dim_; }
    const void* GetTensor() const { return tensor_; }
    const int64_t* GetIds() const { return ids_; }
    const float* GetDistance() const { return dist_; }
    const size_t* GetLims() const { return lims_; }
    // keyed values (dataset.h:423-441); the one key this library reads is meta::EMB_LIST_OFFSET (const size_t*)
    template <typename T> void Set(const std::string& k, T v) { kv_[k] = (const void*)v; }
    template <typename T> T Get(const std::string& k) const {
        auto it = kv_.find(k);
        return it == kv_.end() ? T() : (T)it->second;
    }
 private:
    std::map<std::string, const void*> kv_;
    int64_t rows_ = 0, dim_ = 0;
    const void* tensor_ = nullptr;
    const int64_t* ids_ = nullptr;
    const float* dist_ = nullptr;
    const size_t* lims_ = nullptr;
    bool is_owner_ = true, owned_tensor_ = false;
    std::string json_info_;
};
using DataSetPtr = std::shared_ptr<DataSet>;

// borrows `tensor` (dataset.h:452-459: is_owner=false)
inline DataSetPtr GenDataSet(int64_t rows, int64_t dim, const void* tensor) {
    auto d = std::make_shared<DataSet>();
    d->SetRows(rows); d->SetDim(dim); d->SetTensor(tensor); d->SetIsOwner(false);
    return d;
}
// takes ownership of new[]-allocated ids/dist (dataset.h:499-524); dim == k
inline DataSetPtr GenResultDataSet(int64_t nq, int64_t topk, const int64_t* ids, const float* dist) {
    auto d = std::make_shared<DataSet>();
    d->SetRows(nq); d->SetDim(topk); d->SetIds(ids); d->SetDistance(dist); d->SetIsOwner(true);
    return d;
}
inline DataSetPtr GenResultDataSet(int64_t nq, const int64_t* ids, const float* dist, const size_t* lims) {
    auto d = std::make_shared<DataSet>();
    d->SetRows(nq); d->SetIds(ids); d->SetDistance(dist); d->SetLims(lims); d->SetIsOwner(true);
    return d;
}
inline DataSetPtr GenIdsDataSet(int64_t rows, const int64_t* ids) {
    auto d = std::make_shared<DataSet>();
    d->SetRows(rows); d->SetIds(ids); d->SetIsOwner(false);
    return d;
}

// ------------------------------------------------------------------ BitsetView (bit set => filtered out)
// include/knowhere/bitsetview.h:131-175: bit index = out_ids[internal_id + id_offset] when an id map is attached, else
// internal_id + id_offset.  The GPU kernels take a plain bitmap over internal ids, so a view with an offset or an id map
// is materialised once per call (as the in-tree GPU precedent does: src/index/gpu_cuvs/gpu_cuvs.h:139-156).
class BitsetView {
 public:
    BitsetView() = default;
    BitsetView(const uint8_t* data, size_t num_bits) : bits_(data), num_bits_(num_bits), vector_count_(num_bits) {}
    BitsetView(std::nullptr_t) {}
    bool empty() const { return num_bits_ == 0; }
    size_t size() const { return vector_count_; }
    size_t num_bits() const { return num_bits_; }
    const uint8_t* data() const { return bits_; }
    void set_vector_count(size_t n) { vector_count_ = n; }
    void set_id_offset(size_t o) { id_offset_ = o; }
    size_t id_offset() const { return id_offset_; }
    void set_out_ids(const int64_t* out_ids, size_t count) { out_ids_ = out_ids; out_ids_count_ = count; }
    bool has_out_ids() const { return out_ids_count_ != 0; }
    bool is_plain() const { return id_offset_ == 0 && out_ids_count_ == 0; }
    // true when backend (internal) id `index` is to be skipped
    bool test(int64_t index) const {
        if (index < 0) return true;
        size_t out_id = (size_t)index + id_offset_;
        if (has_out_ids()) {
            if (out_id >= out_ids_count_) return true;
            const int64_t mapped = out_ids_[out_id];
            if (mapped < 0) return true;
            out_id = (size_t)mapped;
        }
        if (out_id >= num_bits_) return true;
        return (bits_[out_id >> 3] >> (out_id & 7)) & 1;
    }
    // plain bitmap over internal ids [0, n)
    std::vector<uint8_t> materialize(size_t n) const {
        std::vector<uint8_t> out((n + 7) / 8, 0);
        for (size_t i = 0; i < n; i++)
            if (test((int64_t)i)) out[i >> 3] |= (uint8_t)(1u << (i & 7));
        return out;
    }
 private:
    const uint8_t* bits_ = nullptr;
    size_t num_bits_ = 0, vector_count_ = 0, id_offset_ = 0;
    const int64_t* out_ids_ = nullptr;
    size_t out_ids_count_ = 0;
};

// ------------------------------------------------------------------ BinarySet
struct Binary { std::shared_ptr<uint8_t[]> data; int64_t size = 0; };
using BinaryPtr = std::shared_ptr<Binary>;
class BinarySet {
 public:
    BinaryPtr GetByName(const std::string& n) const { auto it = m_.find(n); return it == m_.end() ? nullptr : it->second; }
    void Append(const std::string& n, std::shared_ptr<uint8_t[]> data, int64_t size) {
        auto b = std::make_shared<Binary>(); b->data = std::move(data); b->size = size; m_[n] = b;
    }
    bool Contains(const std::string& n) const { return m_.count(n) != 0; }
 private:
    std::map<std::string, BinaryPtr> m_;
};

struct fp32 {};  // data-type tag (include/knowhere/operands.h); this library serves fp32

// ------------------------------------------------------------------ IndexNode over the C ABI
class IndexNode {
 public:
    // IndexNode::iterator (index_node.h:69-88): results in best-first order, one at a time
    class iterator {
     public:
        virtual ~iterator() = default;
        virtual expected<std::pair<int64_t, float>> Next() noexcept = 0;
        virtual expected<bool> HasNext() noexcept = 0;
    };
    using IteratorPtr = std::shared_ptr<iterator>;
    virtual ~IndexNode() = default;
    virtual Status Train(const DataSetPtr ds, const Json& cfg) = 0;
    virtual Status Add(const DataSetPtr ds, const Json& cfg) = 0;
    virtual Status Build(const DataSetPtr ds, const Json& cfg) {  // index_node.h:100-104: Train + Add
        Status s = Train(ds, cfg);
        return s != Status::success ? s : Add(ds, cfg);
    }
    virtual expected<DataSetPtr> Search(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const = 0;
    virtual expected<DataSetPtr> RangeSearch(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const = 0;
    virtual expected<DataSetPtr> GetVectorByIds(const DataSetPtr ds) const = 0;
    virtual bool HasRawData(const std::string& metric_type) const = 0;
    virtual Status Serialize(BinarySet& bs) const = 0;
    virtual Status Deserialize(const BinarySet& bs, const Json& cfg) = 0;
    virtual Status DeserializeFromFile(const std::string& filename, const Json& cfg) = 0;
    virtual expected<DataSetPtr> GetIndexMeta(const Json& cfg) const = 0;
    virtual expected<std::vector<IteratorPtr>> AnnIterator(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const = 0;
    virtual int64_t Dim() const = 0;
    virtual int64_t Size() const = 0;
    virtual int64_t Count() const = 0;
    virtual std::string Type() const = 0;
};

inline int kb2_metric_of(const Json& cfg, Status& st) {
    const std::string m = cfg.get_string(meta::METRIC_TYPE, "L2");
    st = Status::success;
    if (m == "L2") return KB2_METRIC_L2;
    if (m == "IP") return KB2_METRIC_IP;
    if (m == "COSINE") return KB2_METRIC_COSINE;
    st = Status::invalid_metric_type;
    return -1;
}

// emb-list metric names (emb_list_utils.h:225-263, case-insensitive as IsMetricType): true for every MAX_SIM* name, with
// `code` the C ABI metric, or -1 for MAX_SIM_HAMMING / MAX_SIM_JACCARD (no binary vectors here)
inline bool kb2_emb_list_metric(const std::string& name, int& code) {
    std::string m = name;
    for (auto& c : m) c = (char)toupper((unsigned char)c);
    if (m == metric::MAX_SIM || m == metric::MAX_SIM_COSINE) code = KB2_METRIC_MAX_SIM_COSINE;
    else if (m == metric::MAX_SIM_IP) code = KB2_METRIC_MAX_SIM_IP;
    else if (m == metric::MAX_SIM_L2) code = KB2_METRIC_MAX_SIM_L2;
    else if (m == metric::MAX_SIM_HAMMING || m == metric::MAX_SIM_JACCARD) code = -1;
    else return false;
    return true;
}
// The lists of an EMB_LIST_OFFSET over `rows` rows, as EmbListOffset(lims, rows) reads them (emb_list_utils.h:30-41):
// offsets up to the first one equal to the row count, so trailing empty lists are dropped.  False when no offset equals it.
inline bool kb2_emb_list_offsets(const size_t* lims, int64_t rows, std::vector<int64_t>& out) {
    out.clear();
    size_t i = 0;
    for (; (int64_t)lims[i] < rows; i++) out.push_back((int64_t)lims[i]);
    out.push_back((int64_t)lims[i]);
    return (int64_t)lims[i] == rows;
}

class B200IndexNode : public IndexNode {
 public:
    explicit B200IndexNode(std::string type, int device = 0) : type_(std::move(type)), device_(device) {}
    ~B200IndexNode() override { if (h_) kb2_index_destroy(h_); }

    Status Train(const DataSetPtr ds, const Json& cfg) override {
        if (!ds) return Status::invalid_args;
        if (!h_) {
            Status st;
            const int metric = kb2_metric_of(cfg, st);
            if (st != Status::success) return st;
            int rc = kb2_index_create(type_.c_str(), metric, (int)ds->GetDim(), cfg.dump().c_str(), device_, &h_);
            if (rc) return (Status)rc;
        }
        return (Status)kb2_index_train(h_, (const float*)ds->GetTensor(), ds->GetRows());
    }
    Status Add(const DataSetPtr ds, const Json&) override {
        if (!h_) return Status::index_not_trained;
        return (Status)kb2_index_add(h_, (const float*)ds->GetTensor(), ds->GetRows(), nullptr);
    }
    // Build with EMB_LIST_OFFSET and a MAX_SIM metric (index_node.cc:453-507): the handle over every row with the sub-metric
    // (MAX_SIM_L2 -> L2, MAX_SIM_IP -> IP, MAX_SIM / MAX_SIM_COSINE -> COSINE), then the document offsets.  TokenANN (the
    // default) indexes the rows; with "emb_list_strategy": "muvera" the handle keeps them and the offsets build the base
    // over the documents' encodings.
    Status Build(const DataSetPtr ds, const Json& cfg) override {
        if (!ds) return Status::invalid_args;
        int code = 0;
        const bool el_metric = kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code);
        const size_t* lims = ds->Get<const size_t*>(meta::EMB_LIST_OFFSET);
        if (!el_metric && !lims) return IndexNode::Build(ds, cfg);
        if (!el_metric || !lims) return Status::emb_list_inner_error;
        if (code < 0) return Status::invalid_metric_type;
        std::vector<int64_t> xl;
        if (!kb2_emb_list_offsets(lims, ds->GetRows(), xl)) return Status::invalid_args;
        Json sub = cfg;
        sub[meta::METRIC_TYPE] = code == KB2_METRIC_MAX_SIM_L2 ? metric::L2 : code == KB2_METRIC_MAX_SIM_IP ? metric::IP : metric::COSINE;
        const Status s = IndexNode::Build(ds, sub);
        if (s != Status::success) return s;
        const int rc = kb2_index_set_emb_list(h_, xl.data(), (int64_t)xl.size() - 1, code);
        if (rc) return (Status)rc;
        el_metric_ = code;
        muvera_ = cfg.get_string(meta::EMB_LIST_STRATEGY, meta::EMB_LIST_STRATEGY_TOKENANN) == meta::EMB_LIST_STRATEGY_MUVERA;
        return Status::success;
    }
    // plain internal-id bitmap for the C ABI (a view with an id offset / id map is materialised)
    struct PlainBits {
        std::vector<uint8_t> store;
        const uint8_t* data = nullptr;
        int64_t nbits = 0;
    };
    // n: ids the bitmap covers (rows, or documents of an emb-list search; < 0: the index's rows)
    PlainBits plain_bits(const BitsetView& bitset, int64_t n = -1) const {
        PlainBits p;
        if (bitset.empty()) return p;
        if (bitset.is_plain()) { p.data = bitset.data(); p.nbits = (int64_t)bitset.num_bits(); return p; }
        if (n < 0) n = kb2_index_count(h_);
        p.store = bitset.materialize((size_t)n);
        p.data = p.store.data();
        p.nbits = n;
        return p;
    }
    // index_node.cc:275-297: a MAX_SIM metric needs query list offsets and the reverse; both go to the emb-list search
    expected<DataSetPtr> Search(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const override {
        if (!h_) return expected<DataSetPtr>::Err(Status::empty_index, "index not loaded");
        int code = 0;
        const bool el_metric = kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code);
        const size_t* ql = ds->Get<const size_t*>(meta::EMB_LIST_OFFSET);
        if (el_metric && !ql)
            return expected<DataSetPtr>::Err(Status::emb_list_inner_error,
                                             "Not found emb_list offset in query dataset, but metric type is of emb_list");
        if (!el_metric && ql)
            return expected<DataSetPtr>::Err(Status::emb_list_inner_error,
                                             "Invalid emb_list metric type, but found emb_list offset in query dataset.");
        if (el_metric) return SearchEmbList(ds, cfg, bitset, ql, code);
        const int64_t nq = ds->GetRows();
        const int k = cfg.get<int>(meta::TOPK, 0);
        if (k <= 0) return expected<DataSetPtr>::Err(Status::invalid_args, "k must be positive");
        auto ids = std::make_unique<int64_t[]>(nq * k);   // index.cc: ids/dist = new[rows*k] (ivf.cc:913-914)
        auto dis = std::make_unique<float[]>(nq * k);
        const PlainBits pb = plain_bits(bitset);
        int rc = kb2_index_search(h_, (const float*)ds->GetTensor(), nq, k, cfg.dump().c_str(), pb.data, pb.nbits, ids.get(),
                                  dis.get());
        if (rc) return expected<DataSetPtr>::Err((Status)rc, kb2_last_error());
        return GenResultDataSet(nq, k, ids.release(), dis.release());
    }
    // TokenANN search (emb_list_strategy_token_ann.cc:51-175): one result row per query list, ids are documents; the bitset
    // addresses documents
    expected<DataSetPtr> SearchEmbList(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset, const size_t* ql,
                                       int code) const {
        if (code < 0 || (el_metric_ >= 0 && code != el_metric_))
            return expected<DataSetPtr>::Err(Status::invalid_metric_type, "emb_list metric differs from the index's");
        const int k = cfg.get<int>(meta::TOPK, 0);
        if (k <= 0) return expected<DataSetPtr>::Err(Status::invalid_args, "k must be positive");
        std::vector<int64_t> lims;
        if (!kb2_emb_list_offsets(ql, ds->GetRows(), lims))
            return expected<DataSetPtr>::Err(Status::invalid_args, "emb_list offsets do not end at the row count");
        const int64_t n_lists = (int64_t)lims.size() - 1;
        int64_t n_docs = 0;
        if (kb2_index_emb_list_offsets(h_, &n_docs, nullptr) != 0)
            return expected<DataSetPtr>::Err(Status::emb_list_inner_error, "emb_list offset not initialized");
        auto ids = std::make_unique<int64_t[]>(std::max<int64_t>(n_lists * k, 1));
        auto dis = std::make_unique<float[]>(std::max<int64_t>(n_lists * k, 1));
        const PlainBits pb = plain_bits(bitset, n_docs);
        const int rc = kb2_index_search_emb_list(h_, (const float*)ds->GetTensor(), lims.data(), n_lists, k, cfg.dump().c_str(),
                                                 pb.data, pb.nbits, ids.get(), dis.get(), nullptr);
        if (rc) return expected<DataSetPtr>::Err((Status)rc, kb2_last_error());
        return GenResultDataSet(n_lists, k, ids.release(), dis.release());
    }
    expected<DataSetPtr> RangeSearch(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const override {
        if (!h_) return expected<DataSetPtr>::Err(Status::empty_index, "index not loaded");
        int code = 0;
        if (kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code))   // index_node.cc:301-310
            return expected<DataSetPtr>::Err(Status::emb_list_inner_error, "range search is not supported for emb_list");
        if (!cfg.contains(meta::RADIUS)) return expected<DataSetPtr>::Err(Status::invalid_args, "radius missing");
        const int64_t nq = ds->GetRows();
        int64_t *lims = nullptr, *ids = nullptr;
        float* dist = nullptr;
        const bool has_rf = cfg.contains(meta::RANGE_FILTER);
        const PlainBits pb = plain_bits(bitset);
        int rc = kb2_index_range_search(h_, (const float*)ds->GetTensor(), nq, cfg.get<float>(meta::RADIUS, 0.f),
                                        cfg.get<float>(meta::RANGE_FILTER, 0.f), has_rf ? 1 : 0, cfg.dump().c_str(),
                                        pb.data, pb.nbits, &lims, &ids, &dist);
        if (rc) return expected<DataSetPtr>::Err((Status)rc, kb2_last_error());
        const int64_t tot = lims[nq];
        auto o_l = new size_t[nq + 1];
        auto o_i = new int64_t[tot > 0 ? tot : 1];
        auto o_d = new float[tot > 0 ? tot : 1];
        for (int64_t i = 0; i <= nq; i++) o_l[i] = (size_t)lims[i];
        memcpy(o_i, ids, tot * 8);
        memcpy(o_d, dist, tot * 4);
        kb2_free(lims); kb2_free(ids); kb2_free(dist);
        return GenResultDataSet(nq, o_i, o_d, o_l);
    }
    expected<DataSetPtr> GetVectorByIds(const DataSetPtr ds) const override {
        if (!h_) return expected<DataSetPtr>::Err(Status::empty_index, "index not loaded");
        const int64_t n = ds->GetRows(), d = kb2_index_dim(h_);
        auto out = new float[n * d];
        int rc = kb2_index_get_vector_by_ids(h_, ds->GetIds(), n, out);
        if (rc) { delete[] out; return expected<DataSetPtr>::Err((Status)rc, kb2_last_error()); }
        auto r = std::make_shared<DataSet>();
        r->SetRows(n); r->SetDim(d); r->SetTensor(out); r->SetIsOwner(true); r->SetOwnedTensor(true);
        return r;
    }
    bool HasRawData(const std::string&) const override { return h_ && kb2_index_has_raw_data(h_); }
    // Serialize: ONE binary named after the index type holding the faiss fourcc stream, exactly what the reference's
    // nodes write (flat.cc:323-343, ivf.cc:1717-1741, faiss_hnsw.cc:188-217), so the reference's CPU nodes can load it.
    // Indexes the wire format cannot express (COSINE keeps unit vectors only; custom ids; GPU_CAGRA) use the "KB2I" container.
    Status Serialize(BinarySet& bs) const override {
        if (!h_) return Status::empty_index;
        uint8_t* p = nullptr; size_t n = 0;
        // GPU_CAGRA keeps its own type and build parameters in the container (its graph as an HNSW stream is
        // kb2_index_serialize_faiss, for the reference's CPU HNSW node)
        const bool cagra = type_ == "GPU_CAGRA" || type_ == "GPU_CUVS_CAGRA";
        int rc = cagra ? KB2_NOT_IMPLEMENTED : kb2_index_serialize_faiss(h_, &p, &n);
        if (rc == KB2_NOT_IMPLEMENTED) rc = kb2_index_serialize(h_, &p, &n);
        if (rc) return (Status)rc;
        std::shared_ptr<uint8_t[]> buf(new uint8_t[n]);
        memcpy(buf.get(), p, n);
        kb2_free(p);
        bs.Append(type_, buf, (int64_t)n);
        // a MUVERA index's "KB2I" blob holds its strategy, parameters, offsets and token rows itself
        if (el_metric_ < 0 || muvera_) return Status::success;
        // EMB_LIST_META (index_node.cc:527-597, emb_list_strategy_token_ann.cc:176-192): [int64 "ELMF_V2"][size_t type
        // length]["tokenann"][int32 "TOKA"][int32 1][size_t count][size_t offsets[count]]
        int64_t n_docs = 0;
        int rc2 = kb2_index_emb_list_offsets(h_, &n_docs, nullptr);
        if (rc2) return (Status)rc2;
        std::vector<int64_t> lims((size_t)n_docs + 1);
        rc2 = kb2_index_emb_list_offsets(h_, &n_docs, lims.data());
        if (rc2) return (Status)rc2;
        const std::string type = meta::EMB_LIST_STRATEGY_TOKENANN;
        const size_t type_len = type.size(), count = lims.size();
        const int64_t size = 8 + 8 + (int64_t)type_len + 4 + 4 + 8 + 8 * (int64_t)count;
        std::shared_ptr<uint8_t[]> mb(new uint8_t[size]);
        uint8_t* w = mb.get();
        auto put = [&](const void* v, size_t len) { memcpy(w, v, len); w += len; };
        const int64_t magic = kEmbListMetaMagic;
        const int32_t toka = kTokenAnnMagic, version = 1;
        put(&magic, 8); put(&type_len, 8); put(type.data(), type_len); put(&toka, 4); put(&version, 4); put(&count, 8);
        for (int64_t v : lims) { const size_t u = (size_t)v; put(&u, 8); }
        bs.Append(meta::EMB_LIST_META, mb, size);
        return Status::success;
    }
    // With EMB_LIST_META the emb-list metric comes from cfg, as in index_node.cc:599-657; the meta is ELMF_V2 (its TokenANN
    // blob TOKA v1 or the legacy layout) or the legacy [size_t count][size_t offsets] alone.
    Status Deserialize(const BinarySet& bs, const Json& cfg) override {
        auto b = bs.GetByName(type_);
        if (!b) return Status::invalid_binary_set;
        auto mb = bs.GetByName(meta::EMB_LIST_META);
        int code = -1;
        if (mb && (!kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, ""), code) || code < 0)) return Status::invalid_metric_type;
        if (h_) { kb2_index_destroy(h_); h_ = nullptr; }
        el_metric_ = -1;
        muvera_ = false;
        uint32_t magic = 0;
        if (b->size >= 4) memcpy(&magic, b->data.get(), 4);
        const int rc = magic == 0x4932424b ? kb2_index_deserialize(b->data.get(), (size_t)b->size, device_, &h_)
                                           : kb2_index_deserialize_faiss(b->data.get(), (size_t)b->size, 0, device_, &h_);
        if (rc || !mb) return (Status)rc;
        std::vector<int64_t> lims;
        if (!parse_emb_list_meta(mb->data.get(), mb->size, lims)) return Status::emb_list_inner_error;
        const int rc2 = kb2_index_set_emb_list(h_, lims.data(), (int64_t)lims.size() - 1, code);
        if (rc2) return (Status)rc2;
        el_metric_ = code;
        return Status::success;
    }
    static constexpr int64_t kEmbListMetaMagic = 0x454C4D465F563200LL;   // "ELMF_V2\0" (emb_list_strategy.h:291)
    static constexpr int32_t kTokenAnnMagic = 0x544F4B41;                // "TOKA"
    // the document offsets of an EMB_LIST_META blob; false when it is malformed or names another strategy
    static bool parse_emb_list_meta(const uint8_t* p, int64_t size, std::vector<int64_t>& lims) {
        int64_t o = 0;
        auto rd = [&](void* dst, int64_t len) {
            if (len < 0 || o + len > size) return false;
            memcpy(dst, p + o, (size_t)len);
            o += len;
            return true;
        };
        int64_t magic = 0;
        if (size >= 8) memcpy(&magic, p, 8);
        if (magic == kEmbListMetaMagic) {
            o = 8;
            size_t type_len = 0;
            if (!rd(&type_len, 8) || type_len > (size_t)(size - o)) return false;
            if (std::string((const char*)p + o, type_len) != meta::EMB_LIST_STRATEGY_TOKENANN) return false;
            o += (int64_t)type_len;
            int32_t toka = 0;
            if (o + 4 <= size) memcpy(&toka, p + o, 4);
            if (toka == kTokenAnnMagic) {
                int32_t version = 0;
                o += 4;
                if (!rd(&version, 4) || version > 1) return false;
            }
        }
        size_t count = 0;
        if (!rd(&count, 8) || count < 2 || count > (size_t)(size - o) / 8) return false;
        lims.resize(count);
        for (size_t i = 0; i < count; i++) {
            size_t v = 0;
            rd(&v, 8);
            lims[i] = (int64_t)v;
        }
        return true;
    }
    Status DeserializeFromFile(const std::string& filename, const Json&) override {
        if (h_) { kb2_index_destroy(h_); h_ = nullptr; }
        return (Status)kb2_index_deserialize_from_file(filename.c_str(), device_, &h_);
    }
    expected<DataSetPtr> GetIndexMeta(const Json&) const override {
        if (!h_) return expected<DataSetPtr>::Err(Status::empty_index, "index not loaded");
        char buf[1024];
        int rc = kb2_index_get_meta(h_, buf, sizeof(buf));
        if (rc) return expected<DataSetPtr>::Err((Status)rc, kb2_last_error());
        auto r = std::make_shared<DataSet>();
        r->SetJsonInfo(buf);
        return r;
    }
    // AnnIterator (index.h:187-195, index_node.h:1099-1200): one iterator per query yielding (id, distance) best-first.
    // Backed by batched searches with a doubling k (64, 128, ... up to 16384, the largest k FLAT, IVF and HNSW searches
    // accept; on HNSW ef = k): results are a deterministic prefix-stable order, so the iterator resumes where the previous
    // batch ended.
    class SearchIterator : public iterator {
     public:
        SearchIterator(const B200IndexNode* node, std::vector<float> q, Json cfg, PlainBits bits)
            : node_(node), q_(std::move(q)), cfg_(std::move(cfg)), bits_(std::move(bits)) {
            if (!bits_.store.empty()) bits_.data = bits_.store.data();
        }
        expected<bool> HasNext() noexcept override {
            skip_seen();
            if (pos_ < ids_.size() && ids_[pos_] >= 0) return true;
            if (exhausted_) return false;
            refill();
            skip_seen();
            return pos_ < ids_.size() && ids_[pos_] >= 0;
        }
        expected<std::pair<int64_t, float>> Next() noexcept override {
            auto h = HasNext();
            if (!h.has_value() || !h.value()) return expected<std::pair<int64_t, float>>::Err(Status::invalid_args, "iterator exhausted");
            auto r = std::make_pair(ids_[pos_], dis_[pos_]);
            seen_.insert(ids_[pos_]);
            pos_++;
            return r;
        }
     private:
        // a larger batch repeats the earlier results (exactly for FLAT / IVF; a graph search with a larger beam may reorder a
        // few of them): never hand out an id twice
        void skip_seen() {
            while (pos_ < ids_.size() && ids_[pos_] >= 0 && seen_.count(ids_[pos_])) pos_++;
        }
        void refill() {
            pos_ = 0;
            const int64_t count = kb2_index_count(node_->h_);
            const int next_k = (int)std::min<int64_t>(std::min<int64_t>(count, kMaxIteratorK), k_ == 0 ? 64 : 2 * (int64_t)k_);
            if (next_k <= k_) { exhausted_ = true; return; }
            k_ = next_k;
            ids_.assign(k_, -1);
            dis_.assign(k_, 0.f);
            Json c = cfg_;
            c[indexparam::EF] = std::max<int>(k_, c.get<int>(indexparam::EF, 0));
            int rc = kb2_index_search(node_->h_, q_.data(), 1, k_, c.dump().c_str(), bits_.data, bits_.nbits, ids_.data(), dis_.data());
            if (rc) { exhausted_ = true; ids_.clear(); return; }
            if (k_ >= std::min<int64_t>(count, kMaxIteratorK)) exhausted_ = true;   // nothing larger can be asked for
        }
        static constexpr int64_t kMaxIteratorK = 16384;
        const B200IndexNode* node_;
        std::vector<float> q_;
        Json cfg_;
        PlainBits bits_;
        std::vector<int64_t> ids_;
        std::vector<float> dis_;
        std::set<int64_t> seen_;
        size_t pos_ = 0;
        int k_ = 0;
        bool exhausted_ = false;
    };
    expected<std::vector<IteratorPtr>> AnnIterator(const DataSetPtr ds, const Json& cfg, const BitsetView& bitset) const override {
        if (!h_) return expected<std::vector<IteratorPtr>>::Err(Status::empty_index, "index not loaded");
        if (type_ == "GPU_CAGRA" || type_ == "GPU_CUVS_CAGRA")   // as the reference's GPU nodes (gpu_cuvs.h)
            return expected<std::vector<IteratorPtr>>::Err(Status::not_implemented, "AnnIterator is not supported on GPU_CAGRA");
        int code = 0;
        if (kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code))   // index_node.cc:312-324
            return expected<std::vector<IteratorPtr>>::Err(Status::emb_list_inner_error, "ann iterator is not supported for emb_list");
        const int64_t nq = ds->GetRows(), d = ds->GetDim();
        std::vector<IteratorPtr> out;
        for (int64_t i = 0; i < nq; i++) {
            const float* q = (const float*)ds->GetTensor() + i * d;
            PlainBits pb = plain_bits(bitset);
            if (pb.store.empty() && pb.data) { pb.store.assign(pb.data, pb.data + (pb.nbits + 7) / 8); }   // own a copy: the view may die
            out.push_back(std::make_shared<SearchIterator>(this, std::vector<float>(q, q + d), cfg, std::move(pb)));
        }
        return out;
    }
    int64_t Dim() const override { return h_ ? kb2_index_dim(h_) : 0; }
    int64_t Size() const override { return h_ ? kb2_index_size_bytes(h_) : 0; }
    int64_t Count() const override { return h_ ? kb2_index_count(h_) : 0; }
    std::string Type() const override { return type_; }
    kb2_index_t handle() const { return h_; }
 private:
    std::string type_;
    int device_;
    kb2_index_t h_ = nullptr;
    int el_metric_ = -1;   // KB2_METRIC_MAX_SIM_* of an emb-list index, else -1
    bool muvera_ = false;  // an emb-list index built with the MUVERA strategy
};

// ------------------------------------------------------------------ Index<T> handle (index.h:23-253)
template <typename T1>
class Index {
 public:
    Index() = default;
    explicit Index(std::shared_ptr<T1> n) : node(std::move(n)) {}
    template <typename... Args> static Index<T1> Create(Args&&... a) { return Index<T1>(std::make_shared<T1>(std::forward<Args>(a)...)); }
    Status Build(const DataSetPtr ds, const Json& cfg, bool = true) noexcept { return guard([&] { return node->Build(ds, cfg); }); }
    Status Train(const DataSetPtr ds, const Json& cfg, bool = true) noexcept { return guard([&] { return node->Train(ds, cfg); }); }
    Status Add(const DataSetPtr ds, const Json& cfg, bool = true) noexcept { return guard([&] { return node->Add(ds, cfg); }); }
    expected<DataSetPtr> Search(const DataSetPtr ds, const Json& cfg, const BitsetView& bs, void* = nullptr) const noexcept {
        try { return node->Search(ds, cfg, bs); } catch (const std::exception& e) { return expected<DataSetPtr>::Err(Status::internal_error, e.what()); }
    }
    expected<DataSetPtr> RangeSearch(const DataSetPtr ds, const Json& cfg, const BitsetView& bs, void* = nullptr) const noexcept {
        try { return node->RangeSearch(ds, cfg, bs); } catch (const std::exception& e) { return expected<DataSetPtr>::Err(Status::internal_error, e.what()); }
    }
    expected<DataSetPtr> GetVectorByIds(const DataSetPtr ds, void* = nullptr) const noexcept {
        try { return node->GetVectorByIds(ds); } catch (const std::exception& e) { return expected<DataSetPtr>::Err(Status::internal_error, e.what()); }
    }
    bool HasRawData(const std::string& m) const noexcept { return node->HasRawData(m); }
    Status Serialize(BinarySet& bs) const noexcept { return guard([&] { return node->Serialize(bs); }); }
    Status Deserialize(const BinarySet& bs, const Json& cfg = {}) noexcept { return guard([&] { return node->Deserialize(bs, cfg); }); }
    Status DeserializeFromFile(const std::string& f, const Json& cfg = {}) noexcept { return guard([&] { return node->DeserializeFromFile(f, cfg); }); }
    expected<DataSetPtr> GetIndexMeta(const Json& cfg = {}) const noexcept {
        try { return node->GetIndexMeta(cfg); } catch (const std::exception& e) { return expected<DataSetPtr>::Err(Status::internal_error, e.what()); }
    }
    expected<std::vector<IndexNode::IteratorPtr>> AnnIterator(const DataSetPtr ds, const Json& cfg, const BitsetView& bs, void* = nullptr) const noexcept {
        try { return node->AnnIterator(ds, cfg, bs); } catch (const std::exception& e) { return expected<std::vector<IndexNode::IteratorPtr>>::Err(Status::internal_error, e.what()); }
    }
    int64_t Dim() const noexcept { return node->Dim(); }
    int64_t Size() const noexcept { return node->Size(); }
    int64_t Count() const noexcept { return node->Count(); }
    std::string Type() const noexcept { return node->Type(); }
    T1* Node() const { return node.get(); }
 private:
    template <typename F> static Status guard(F&& f) noexcept {
        try { return f(); } catch (...) { return Status::internal_error; }
    }
    std::shared_ptr<T1> node;
};

// ------------------------------------------------------------------ IndexFactory (index_factory.h:27-72)
class IndexFactory {
 public:
    using Creator = std::function<Index<IndexNode>(const int32_t& version, const void* object)>;
    static IndexFactory& Instance() { static IndexFactory f; return f; }
    template <typename DataType>
    expected<Index<IndexNode>> Create(const std::string& name, const int32_t& version, const void* object = nullptr) {
        auto it = map_.find(name);
        if (it == map_.end())
            return expected<Index<IndexNode>>::Err(Status::invalid_index_error, "index " + name + " not registered");
        if (kb2_device_count() <= 0)   // index_factory.cc:29-45,62-66: GPU index without a device
            return expected<Index<IndexNode>>::Err(Status::cuda_runtime_error, "gpu index is not supported: no sm_90 device");
        return it->second(version, object);
    }
    template <typename DataType>
    const IndexFactory& Register(const std::string& name, Creator c) { map_[name] = std::move(c); return *this; }
 private:
    IndexFactory() {
        for (const char* n : {"FLAT", "IVF_FLAT", "IVF_PQ", "HNSW", "GPU_CAGRA", "GPU_CUVS_CAGRA"}) {
            const std::string name = n;
            map_[name] = [name](const int32_t&, const void*) {
                return Index<IndexNode>(std::static_pointer_cast<IndexNode>(std::make_shared<B200IndexNode>(name)));
            };
        }
    }
    std::map<std::string, Creator> map_;
};

// ------------------------------------------------------------------ BruteForce (brute_force.h:26-69)
class BruteForce {
 public:
    template <typename DataType>
    static expected<DataSetPtr> Search(const DataSetPtr base, const DataSetPtr query, const Json& cfg,
                                       const BitsetView& bitset, void* = nullptr) noexcept {
        int64_t nq = query->GetRows();
        const int k = cfg.get<int>(meta::TOPK, 0);
        if (k <= 0) return expected<DataSetPtr>::Err(Status::invalid_args, "k must be positive");
        int code = 0;
        if (kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code)) {
            // brute_force.cc:270-281: one result row per query list
            const size_t* ql = query->Get<const size_t*>(meta::EMB_LIST_OFFSET);
            if (!ql || !base->Get<const size_t*>(meta::EMB_LIST_OFFSET))
                return expected<DataSetPtr>::Err(Status::invalid_args, "metric type is emb_list, but missing emb_list offset");
            std::vector<int64_t> lims;
            if (!kb2_emb_list_offsets(ql, nq, lims))
                return expected<DataSetPtr>::Err(Status::invalid_args, "emb_list offsets do not end at the row count");
            nq = (int64_t)lims.size() - 1;
        }
        auto ids = std::make_unique<int64_t[]>(nq * k);
        auto dis = std::make_unique<float[]>(nq * k);
        Status s = SearchWithBuf<DataType>(base, query, ids.get(), dis.get(), cfg, bitset);
        if (s != Status::success) return expected<DataSetPtr>::Err(s, kb2_last_error());
        return GenResultDataSet(nq, k, ids.release(), dis.release());
    }
    template <typename DataType>
    static Status SearchWithBuf(const DataSetPtr base, const DataSetPtr query, int64_t* ids, float* dis, const Json& cfg,
                                const BitsetView& bitset, void* = nullptr) noexcept {
        const size_t* bl = base->Get<const size_t*>(meta::EMB_LIST_OFFSET);
        const size_t* ql = query->Get<const size_t*>(meta::EMB_LIST_OFFSET);
        int code = 0;
        if (kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code)) {
            // brute_force.cc:626-665
            if (!bl || !ql) return Status::invalid_metric_type;
            std::vector<int64_t> xl, qlv;
            if (!kb2_emb_list_offsets(bl, base->GetRows(), xl) || !kb2_emb_list_offsets(ql, query->GetRows(), qlv))
                return Status::invalid_args;
            return (Status)kb2_bruteforce_search_emb_list(
                (const float*)base->GetTensor(), xl.data(), (int64_t)xl.size() - 1, (int)base->GetDim(), code,
                (const float*)query->GetTensor(), qlv.data(), (int64_t)qlv.size() - 1, cfg.get<int>(meta::TOPK, 0), bitset.data(),
                (int64_t)bitset.size(), ids, dis, nullptr, 0, nullptr);
        }
        if (ql) return Status::invalid_metric_type;   // brute_force.cc:673-676: emb-list query, single-vector metric
        Status st;
        const int metric = kb2_metric_of(cfg, st);
        if (st != Status::success) return st;
        return (Status)kb2_bruteforce_search((const float*)base->GetTensor(), base->GetRows(), (int)base->GetDim(), metric,
                                             (const float*)query->GetTensor(), query->GetRows(),
                                             cfg.get<int>(meta::TOPK, 0), bitset.data(), (int64_t)bitset.size(), ids, dis,
                                             0, nullptr);
    }
    template <typename DataType>
    static expected<DataSetPtr> RangeSearch(const DataSetPtr base, const DataSetPtr query, const Json& cfg,
                                            const BitsetView& bitset, void* = nullptr) noexcept {
        int code = 0;
        if (kb2_emb_list_metric(cfg.get_string(meta::METRIC_TYPE, "L2"), code))   // index_node.cc:301-310
            return expected<DataSetPtr>::Err(Status::emb_list_inner_error, "range search is not supported for emb_list");
        Status st;
        const int metric = kb2_metric_of(cfg, st);
        if (st != Status::success) return expected<DataSetPtr>::Err(st, "bad metric");
        const int64_t nq = query->GetRows();
        int64_t *lims = nullptr, *ids = nullptr;
        float* dist = nullptr;
        int rc = kb2_bruteforce_range_search((const float*)base->GetTensor(), base->GetRows(), (int)base->GetDim(), metric,
                                             (const float*)query->GetTensor(), nq, cfg.get<float>(meta::RADIUS, 0.f),
                                             cfg.get<float>(meta::RANGE_FILTER, 0.f), cfg.contains(meta::RANGE_FILTER),
                                             bitset.data(), (int64_t)bitset.size(), &lims, &ids, &dist, 0, nullptr);
        if (rc) return expected<DataSetPtr>::Err((Status)rc, kb2_last_error());
        const int64_t tot = lims[nq];
        auto o_l = new size_t[nq + 1];
        auto o_i = new int64_t[tot > 0 ? tot : 1];
        auto o_d = new float[tot > 0 ? tot : 1];
        for (int64_t i = 0; i <= nq; i++) o_l[i] = (size_t)lims[i];
        memcpy(o_i, ids, tot * 8);
        memcpy(o_d, dist, tot * 4);
        kb2_free(lims); kb2_free(ids); kb2_free(dist);
        return GenResultDataSet(nq, o_i, o_d, o_l);
    }
};

}  // namespace knowhere
