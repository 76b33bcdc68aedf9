// kb2_muvera.cuh — the MUVERA emb-list strategy's encoder and index object (the reference's
// src/index/emb_list/emb_list_strategy_muvera.cc, include/knowhere/config.h:636-655,836-855).  DESIGN §4.11.
//
// Each token x is hashed per repeat r into bucket b = sum of 2^p over the projections p with dot(proj[r][p], x) >= 0
// (SimHash, B = 2^P buckets).  A document's Fixed Dimensional Encoding (FDE) is [R][B][d]: per (repeat, bucket) the sum
// of its tokens in that bucket, in token order, scaled by 1 / count when the count is above 1 (mean); a query list's FDE
// is the same sum without the scaling.  Projections come from std::normal_distribution<float>(0, 1) over
// std::mt19937(S + r), drawn on the host with the standard library (kb2_muvera_proj.cpp).
//
//   muvera_bucket_kernel  one CTA per (block of tokens, repeat), the repeat's P x d projections in shared memory, one warp
//                         per token: fp32 fmaf partial dots over strided dimensions, a butterfly sum, the sign test.  At
//                         most 2 * tokens * R * P * d FLOP (1M tokens at R = 7, P = 4, d = 128: 7.2 GFLOP): CUDA cores,
//                         no tensor cores;
//   muvera_encode_kernel  one CTA per (document or list, repeat): each thread owns one dimension of all B buckets in shared
//                         memory (B x 128 floats, 8 KB at B = 16), adds the tokens in token order with one fp32 add per
//                         element (the reference's fvec_madd with factor 1 is an exact add), applies the counts and writes
//                         the repeat's B x d slice of the E = R * B * d row coalesced, zeros included.
// Given the same buckets the FDE is bit-identical to the reference; only a sign test on a dot product within fp32
// rounding of 0 can pick another bucket (the device adds in another order than the reference's SIMD inner product).
//
// MuveraIndex is the handle of an HNSW or IVF_FLAT index created with "emb_list_strategy": "muvera".  kb2_index_add keeps
// the token rows (raw, also under COSINE: the reference encodes raw tokens); kb2_index_set_emb_list encodes every document
// and builds `base`, an index of the same type over the n_docs FDE rows (dimension E); the emb-list search
// (kb2_emb_list_index.cuh) encodes the query lists, searches `base` and re-ranks its documents by exact MaxSim.
#pragma once
#include "kb2_hnsw.cuh"

namespace kb2 {

constexpr int kMuveraDimBlock = 128;   // threads of muvera_encode_kernel: dimensions per pass over a document's tokens

struct MuveraParams {
    int P = 4;    // muvera_num_projections: B = 2^P buckets per repeat
    int R = 7;    // muvera_num_repeats
    int S = 42;   // muvera_seed
};

// [R][P][d] projections (kb2_muvera_proj.cpp, compiled without FMA contraction)
std::vector<float> muvera_projections(int P, int R, int S, int d);
inline std::vector<float>
muvera_projections(const MuveraParams& m, int d) {
    return muvera_projections(m.P, m.R, m.S, d);
}

// bucket[t * R + r] for tokens t < n of x [n][d]
__global__ void __launch_bounds__(256)
muvera_bucket_kernel(const float* __restrict__ x, int64_t n, int d, const float* __restrict__ proj, int P, int R,
                     uint8_t* __restrict__ bucket) {
    extern __shared__ float s_proj[];   // [P][d] of repeat blockIdx.y
    const int r = blockIdx.y;
    for (int i = threadIdx.x; i < P * d; i += blockDim.x) s_proj[i] = proj[(size_t)r * P * d + i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n; t += nwarps) {
        const float* xt = x + t * d;
        uint32_t b = 0;
        for (int p = 0; p < P; p++) {
            float acc = 0.f;
            for (int j = lane; j < d; j += 32) acc = fmaf(s_proj[p * d + j], __ldg(xt + j), acc);
            // butterfly: every lane ends with the same sum (each step adds the same two operands on both partners)
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (acc >= 0.f) b |= 1u << p;
        }
        if (lane == 0) bucket[t * R + r] = (uint8_t)b;
    }
}

// FDE row blockIdx.x (out + blockIdx.x * E) of item i = item0 + blockIdx.x, whose tokens are x / bucket rows
// [lims[i] - lims[item0], lims[i + 1] - lims[item0]); repeat blockIdx.y
__global__ void __launch_bounds__(kMuveraDimBlock)
muvera_encode_kernel(const float* __restrict__ x, const uint8_t* __restrict__ bucket, const int64_t* __restrict__ lims,
                     int64_t item0, int d, int P, int R, bool mean, float* __restrict__ out) {
    extern __shared__ float s_acc[];   // [B][kMuveraDimBlock]: thread j owns column j; then [B] token counts
    const int B = 1 << P, r = blockIdx.y, j = threadIdx.x;
    int* s_cnt = reinterpret_cast<int*>(s_acc + B * kMuveraDimBlock);
    const int64_t it = item0 + blockIdx.x, base = lims[item0];
    const int64_t a = lims[it] - base, e = lims[it + 1] - base;
    if (mean) {
        for (int b = j; b < B; b += blockDim.x) {
            int c = 0;
            for (int64_t t = a; t < e; t++) c += bucket[t * R + r] == b;
            s_cnt[b] = c;
        }
        __syncthreads();
    }
    float* acc = s_acc + j;
    float* row = out + (int64_t)blockIdx.x * ((int64_t)R * B * d) + (int64_t)r * B * d;
    for (int j0 = 0; j0 < d; j0 += kMuveraDimBlock) {
        if (j0 + j >= d) break;
        for (int b = 0; b < B; b++) acc[b * kMuveraDimBlock] = 0.f;
        for (int64_t t = a; t < e; t++) acc[bucket[t * R + r] * kMuveraDimBlock] += __ldg(x + t * d + j0 + j);
        for (int b = 0; b < B; b++) {
            float v = acc[b * kMuveraDimBlock];
            if (mean && s_cnt[b] > 1) v *= 1.0f / (float)s_cnt[b];
            row[(int64_t)b * d + j0 + j] = v;
        }
    }
}

// FDE rows [n_items][E] of items item0 .. item0 + n_items - 1 (d_lims: device offsets; x: [ntok][d] device rows of those
// items' tokens, from lims[item0] on; proj: device projections)
inline void
muvera_encode(const MuveraParams& m, int d, const float* proj, const float* x, int64_t ntok, const int64_t* d_lims,
              int64_t item0, int64_t n_items, bool mean, DevBuf<uint8_t>& bucket, float* out, cudaStream_t st) {
    const size_t smem_b = (size_t)m.P * d * 4;
    KB2_REQUIRE(smem_b <= (size_t)kMaxDynSmem, KB2_INVALID_ARGS, "MUVERA: muvera_num_projections x dim too large for shared memory");
    if (ntok > 0) {
        bucket.ensure((size_t)ntok * m.R);
        const unsigned gx = (unsigned)std::min<int64_t>((ntok + 7) / 8, (int64_t)num_sms() * 8);
        launch<muvera_bucket_kernel>(dim3(gx, (unsigned)m.R), 256, smem_b, st, x, ntok, d, proj, m.P, m.R, bucket.p);
    }
    if (n_items > 0)
        launch<muvera_encode_kernel>(dim3((unsigned)n_items, (unsigned)m.R), kMuveraDimBlock,
                                     ((size_t)1 << m.P) * (kMuveraDimBlock + 1) * 4, st, x, bucket.p, d_lims, item0, d, m.P, m.R, mean,
                                     out);
    KB2_CUDA_CHECK(cudaGetLastError());
}

// The create keys of the emb-list strategy of an HNSW or IVF_FLAT handle (emb_list_strategy.cc:31-43, config.h:836-855;
// an empty or missing strategy is TokenANN); true for MUVERA
inline bool
muvera_params_of(const JsonObj& cfg, MuveraParams& m) {
    const std::string s = cfg.get_str("emb_list_strategy", "tokenann");
    if (s.empty() || s == "tokenann") return false;
    KB2_REQUIRE(s != "lemur", KB2_NOT_IMPLEMENTED, "emb_list_strategy lemur is not implemented");
    KB2_REQUIRE(s == "muvera", KB2_INVALID_ARGS, "unknown emb_list_strategy " + s + " (tokenann or muvera)");
    const long long P = cfg.get_int("muvera_num_projections", 4), R = cfg.get_int("muvera_num_repeats", 7),
                    S = cfg.get_int("muvera_seed", 42);
    KB2_REQUIRE(P >= 1 && P <= 7, KB2_OUT_OF_RANGE_IN_JSON, "muvera_num_projections out of range (1..7)");
    KB2_REQUIRE(R >= 1 && R <= 32, KB2_OUT_OF_RANGE_IN_JSON, "muvera_num_repeats out of range (1..32)");
    KB2_REQUIRE(S >= INT32_MIN && S <= INT32_MAX, KB2_OUT_OF_RANGE_IN_JSON, "muvera_seed out of the int32 range");
    m = MuveraParams{(int)P, (int)R, (int)S};
    return true;
}

struct MuveraIndex : IndexBase {
    MuveraParams mp;
    JsonObj build_cfg;                 // the create JSON: the base's build keys
    std::unique_ptr<IndexBase> base;   // HNSW or IVF_FLAT over the FDE rows of the documents (dimension E)
    DevBuf<float> tokens, tokens_n;    // token rows as added; under COSINE their normalised copy, which the re-rank reads
    size_t tokens_used = 0;
    DevBuf<float> proj;                // [R][P][d], uploaded at attach
    // search scratch: the encoded query lists of a chunk and their tokens' buckets (the attach's buckets too)
    DevBuf<float> fde;
    DevBuf<uint8_t> bucket;

    int64_t E() const { return (int64_t)mp.R * ((int64_t)1 << mp.P) * dim; }
    // an empty base of the handle's type over E-dimensional rows, on the handle's stream
    std::unique_ptr<IndexBase>
    fresh_base() const {
        std::unique_ptr<IndexBase> b;
        if (type == "HNSW") b = std::make_unique<HnswIndex>();
        else b = std::make_unique<IvfIndex>();
        b->init(type, cosine ? KB2_METRIC_COSINE : metric, (int)E(), device);
        b->configure(build_cfg);
        b->set_stream(stream);
        return b;
    }
    // the base, following the handle's stream (kb2_index_set_stream)
    IndexBase&
    base_index() {
        base->stream = stream;
        return *base;
    }

    void
    configure(const JsonObj& cfg) override {
        muvera_params_of(cfg, mp);
        KB2_REQUIRE(E() <= (1 << 20), KB2_INVALID_ARGS, "MUVERA: encoded dimension muvera_num_repeats x 2^muvera_num_projections x dim above 2^20");
        build_cfg = cfg;
        base = fresh_base();   // checks the base's build keys now
    }
    bool raw_rows_on_entry() const override { return true; }
    void train(const float*, int64_t) override {}   // the base is trained over the encoded documents at the attach
    void
    add(const float* x, int64_t n, const int64_t* ids) override {
        if (n <= 0) return;
        KB2_REQUIRE(count() + n < (1ll << 31), KB2_INVALID_ARGS, "MUVERA: too many token rows (at most 2^31 - 1)");
        labels.append(count(), ids, n, count(), false, stream);   // custom ids are refused at the attach, as for TokenANN
        dev_append(tokens, tokens_used, x, (size_t)n * dim, stream);
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }
    void
    search(const float*, int64_t, int, const JsonObj&, const uint8_t*, int64_t, int64_t*, float*) override {
        throw Error(KB2_EMB_LIST_INNER_ERROR,
                    "a MUVERA index is searched with query list offsets (kb2_index_search_emb_list) once its documents are attached");
    }
    int64_t count() const override { return (int64_t)(tokens_used / std::max(dim, 1)); }
    int64_t size_bytes() const override { return (int64_t)(tokens.bytes() + tokens_n.bytes()) + (base ? base->size_bytes() : 0); }
    bool is_trained() const override { return true; }
    bool has_raw() const override { return false; }
    void
    refuse(Op op) const override {
        KB2_REQUIRE(op != kRangeSearch, KB2_EMB_LIST_INNER_ERROR, "RangeSearch is not supported on an emb-list index");
    }
    bool takes_emb_list() const override { return true; }
    std::pair<const float*, const int32_t*>
    emb_list_rows() override {
        return {cosine ? tokens_n.p : tokens.p, nullptr};
    }
    void
    append_meta(std::string& s) const override {
        if (base) base->append_meta(s);
        s += ", \"emb_list_strategy\": \"muvera\", \"muvera_num_projections\": " + std::to_string(mp.P) +
             ", \"muvera_num_repeats\": " + std::to_string(mp.R) + ", \"muvera_seed\": " + std::to_string(mp.S) +
             ", \"muvera_encoded_dim\": " + std::to_string(E());
    }
    // the "KB2I" container holds the base and then the emb-list section (serialize_index / deserialize_index)
    void save(BlobWriter&) override { throw Error(KB2_INTERNAL_ERROR, "MUVERA: saved through its base"); }
    void load(BlobReader&) override { throw Error(KB2_INTERNAL_ERROR, "MUVERA: loaded through its base"); }
    void
    to_faiss(FaissIndexData&) override {
        throw Error(KB2_NOT_IMPLEMENTED, "faiss stream: a MUVERA emb-list index (its token rows would not survive the stream)");
    }

    // The attach (kb2_index_set_emb_list, after its checks; d_lims: the document offsets on the device): projections,
    // the re-rank's rows and the base, either `loaded` (deserialisation) or built here over the encoded documents
    void
    attach(int64_t n_docs, const int64_t* d_lims, std::unique_ptr<IndexBase> loaded) {
        // the base is built over the documents once: new offsets would need the build keys and every encoding again
        KB2_REQUIRE(!emb_list, KB2_NOT_IMPLEMENTED, "a MUVERA index's documents are attached once (its base is built over them)");
        const int d = dim;
        const std::vector<float> h = muvera_projections(mp, d);
        proj.alloc_exact(h.size());
        KB2_CUDA_CHECK(cudaMemcpyAsync(proj.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice, stream));
        const int64_t n = count();
        if (cosine) {
            tokens_n.alloc_exact((size_t)n * d);
            normalize_rows_kernel<<<grid1d(n * 32, 256), 256, 0, stream>>>(tokens.p, n, d, tokens_n.p);
            KB2_CUDA_CHECK(cudaGetLastError());
        }
        if (loaded) {
            KB2_REQUIRE(loaded->dim == E() && loaded->count() == n_docs, KB2_INVALID_BINARY_SET, "MUVERA: the base does not match its emb-list section");
            base = std::move(loaded);
            base->set_stream(stream);
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            return;
        }
        if (base->count() > 0) base = fresh_base();   // an attach that failed part way left rows in the base
        // device memory: the n_docs x E encodings, then the base's own copy of them (under COSINE the normalised copy
        // replaces the encodings before the base reads them)
        DevBuf<float> enc;
        enc.ensure((size_t)n_docs * E());
        muvera_encode(mp, d, proj.p, tokens.p, n, d_lims, 0, n_docs, true, bucket, enc.p, stream);
        IndexBase& b = base_index();
        const float* x = enc.p;
        if (b.cosine) {
            x = b.normalized(enc.p, n_docs);
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            enc.release();
        }
        b.train(x, n_docs);
        b.add(x, n_docs, nullptr);
        b.s_cos_out.release();
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }
};

}  // namespace kb2
