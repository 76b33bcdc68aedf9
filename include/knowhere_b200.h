/*
 * knowhere_b200.h — C ABI of the H100-native ANN search core (libknowhere_b200.so).
 *
 * This is the drop-in boundary.  Every entry point is plain C (pointers + sizes, no
 * C++/torch types) and names the reference interface it stands in for.  A Knowhere
 * build binds these from an IndexNode subclass exactly like the in-tree GPU precedent
 * binds cuVS through a pimpl (reference: src/index/gpu_cuvs/gpu_cuvs.h:71-316,
 * src/common/cuvs/integration/cuvs_knowhere_index.hpp:28-75); see INTEGRATION.md.
 *
 * Conventions
 *   - Return value is a knowhere::Status integer (reference: include/knowhere/expected.h:34-68);
 *     0 = success.  kb2_last_error() returns the thread-local message of the last failure.
 *   - No exception ever crosses this boundary (reference: GuardedCall, expected.h:408-430).
 *   - Vector / query / output pointers may be HOST or DEVICE pointers; the library detects
 *     which (cudaPointerGetAttributes).  Host buffers are staged through pinned memory and
 *     copied on the index's stream inside the call (that is the end-to-end path);
 *     device buffers are used in place (that is the HBM-resident path).
 *   - Results: k entries per query, best first (L2 ascending, IP descending), ties ordered by
 *     ascending id; missing entries have id -1 and distance +FLT_MAX (L2) / -FLT_MAX (IP)
 *     (reference: F/utils/ordered_key_value.h:54-79, K/impl/HnswSearcher.h:414-428).
 *   - ids are int64 (faiss::idx_t; reference include/knowhere/dataset.h:499-510).
 *   - Bitset: bit i set => row i is filtered OUT (reference include/knowhere/bitsetview.h:166);
 *     byte i/8, bit i%8, host or device pointer, NULL = no filter.
 *   - Search on one handle is thread-safe w.r.t. other searches (internally serialised on the
 *     handle's stream; reference: IndexNodeThreadPoolWrapper, index_node_thread_pool_wrapper.cc:33-44).
 *   - There is NO CPU fallback: with no usable CUDA device every call returns
 *     KB2_CUDA_RUNTIME_ERROR (reference: index_factory.cc:29-45,62-66).
 */
#ifndef KNOWHERE_B200_H
#define KNOWHERE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* knowhere::Status values used by this library (expected.h:34-68) */
enum {
    KB2_SUCCESS = 0,
    KB2_INVALID_ARGS = 1,
    KB2_INVALID_PARAM_IN_JSON = 2,
    KB2_OUT_OF_RANGE_IN_JSON = 3,
    KB2_INVALID_METRIC_TYPE = 5,
    KB2_EMPTY_INDEX = 6,
    KB2_NOT_IMPLEMENTED = 7,
    KB2_INDEX_NOT_TRAINED = 8,
    KB2_INDEX_ALREADY_TRAINED = 9,
    KB2_MALLOC_ERROR = 13,
    KB2_INVALID_VALUE_IN_JSON = 16,
    KB2_INVALID_BINARY_SET = 19,
    KB2_CUDA_RUNTIME_ERROR = 22,
    KB2_INTERNAL_ERROR = 27,
    KB2_EMB_LIST_INNER_ERROR = 31
};

/* metric ids (reference: include/knowhere/comp/index_param.h metric names "L2","IP","COSINE"; the MAX_SIM_* emb-list
 * metrics, index_param.h:280-285, only for kb2_bruteforce_search_emb_list and kb2_index_set_emb_list; "MAX_SIM" is
 * MAX_SIM_COSINE; "BM25" only for sparse rows, with IP) */
enum {
    KB2_METRIC_L2 = 0, KB2_METRIC_IP = 1, KB2_METRIC_COSINE = 2,
    KB2_METRIC_MAX_SIM_L2 = 3, KB2_METRIC_MAX_SIM_IP = 4, KB2_METRIC_MAX_SIM_COSINE = 5,
    KB2_METRIC_BM25 = 6
};

typedef struct kb2_index* kb2_index_t;
typedef struct kb2_comm* kb2_comm_t;

/* ---- library ------------------------------------------------------------------------- */
const char* kb2_version(void);
const char* kb2_last_error(void);
/* number of visible CUDA devices with compute capability 10.x; <=0 => library unusable */
int kb2_device_count(void);

/* ---- index lifecycle ------------------------------------------------------------------
 * Replaces IndexFactory::Create<fp32>(name, version) + IndexNode ctor
 * (reference: include/knowhere/index/index_factory.h:27-72, src/index/index_factory.cc:48-86).
 * index_type: "FLAT" | "IVF_FLAT" | "IVF_PQ" | "HNSW"    (index_param.h:27-46)
 * json_cfg  : build-time keys of the reference configs: metric_type, dim, nlist, m, nbits,
 *             refine, refine_type ("flat"|"fp32"), M, efConstruction.  metric KB2_METRIC_COSINE: vectors are
 *             L2-normalised on entry and queries at search (then inner product); HasRawData is false.
 *             (ivf_config.h:25-128, base_hnsw_config.h:36-62).  May be NULL/"" for defaults.
 * "GPU_CAGRA" | "GPU_CUVS_CAGRA" (DESIGN §4.12): a fixed-degree graph built on the device at kb2_index_add (train is a
 *             no-op) and searched by a batched itopk kernel.  Metrics L2, IP, COSINE.  Build keys
 *             intermediate_graph_degree (1..1007, default 128) and graph_degree (1..256, <= the former, default 64),
 *             else KB2_OUT_OF_RANGE_IN_JSON.  The intermediate graph is the exact k-NN graph, or with build_algo
 *             "NN_DESCENT" (any case) the NN-descent graph, nn_descent_niter (1..1000, default 20, else
 *             KB2_OUT_OF_RANGE_IN_JSON) its iteration cap; any other build_algo builds the exact graph.
 *             cache_dataset_on_device and adapt_for_cpu are accepted and have no effect.  Search keys
 *             itopk_size (default max(k, 64), rounded up to a multiple of 32, <= 1024), search_width (default
 *             max(ceil(k / 32), 1)), max_iterations (0: until no pool entry is unexpanded), num_random_samplings
 *             (default 1); max(itopk_size, 32 * search_width) >= k and search_width * graph_degree <= 4096, else
 *             KB2_OUT_OF_RANGE_IN_JSON.  The other cuVS search keys (team_size, thread_block_size, hashmap_*,
 *             persistent, search_algo, max_queries, min_iterations, refine_ratio) and ef are accepted without effect.
 *             Distances are exact fp32.  The graph search serves k <= 1024; HNSW's exact branch (>= 93 % filtered,
 *             or k >= n_valid / 2) serves k <= 16384, and a row with fewer than k results is completed by it.  A
 *             second add, custom ids and sharding return KB2_NOT_IMPLEMENTED, as does RangeSearch;
 *             kb2_index_set_emb_list returns KB2_INVALID_METRIC_TYPE.  kb2_hnsw_export returns the graph as one
 *             HNSW level (levels 1, cum {0, degree}, entry point 0), kb2_hnsw_last_stats {rows evaluated, parents
 *             expanded}, and kb2_index_serialize_faiss an "IHNf" stream the reference's CPU HNSW node loads.
 * "SPARSE_INVERTED_INDEX" | "SPARSE_WAND" (DESIGN §4.13): sparse float rows (kb2_index_add_sparse), metric IP or BM25
 *             (else KB2_INVALID_METRIC_TYPE); dim is ignored and kb2_index_dim returns 0.  Build keys as
 *             sparse_index_node.cc:121-126 and sparse_index_config.h:173-205: BM25 needs bm25_k1 (0..3), bm25_b (0..1)
 *             and bm25_avgdl (>= 0) (missing: KB2_INVALID_ARGS, out of range: KB2_OUT_OF_RANGE_IN_JSON);
 *             inverted_index_algo must be one of the reference's six names (any case) and quant_type fp16 / fp32 (IP)
 *             or u16 / u32 (BM25), else KB2_INVALID_ARGS.  drop_ratio_build, inverted_index_codec, block_max_block_size
 *             and sindi_window_size are accepted without effect: values stay fp32 and every search is exhaustive and
 *             exact, the same for both types and every algorithm.  The dense train / add / search / range search
 *             return KB2_INVALID_ARGS naming the sparse entry point; sharding, emb-lists, GetVectorByIds and the faiss
 *             stream KB2_NOT_IMPLEMENTED.  HasRawData is 0, IsTrained 1; the meta JSON adds sparse_dim and nnz.
 *             kb2_index_size_bytes counts the device postings and term table and the host copy of the rows. */
int kb2_index_create(const char* index_type, int metric, int dim, const char* json_cfg, int device,
                     kb2_index_t* out);
void kb2_index_destroy(kb2_index_t h);

/* run all of this handle's work on an externally owned cudaStream_t (e.g. torch's current
 * stream) so that callers can bracket it with their own CUDA events.  0 = legacy default stream. */
int kb2_index_set_stream(kb2_index_t h, void* cuda_stream);

/* Multi-GPU list/row sharding (SURVEY §8e).  Must be called before train/add/import.
 * IVF_*: every inverted list lives on exactly one rank (greedy size-balanced packing over the global list sizes,
 * identical on all ranks).  FLAT: row i is kept by rank
 * floor(i * world / n) at add time.  HNSW: graph partitions — every rank builds an independent sub-graph over its
 * contiguous row slice of the (single) add() call and all of them are searched with the same ef (SURVEY §8e option 2;
 * recall >= the single graph's in practice, at world x the distance evaluations).
 * Without a communicator Search returns this shard's local top-k (merge shards with kb2_merge_topk after an
 * all-gather); with kb2_index_set_comm the gather + merge happen inside Search. */
int kb2_index_set_shard(kb2_index_t h, int rank, int world);

/* IndexNode::Train (reference: include/knowhere/index/index_node.h:131, ivf.cc:545-807):
 * k-means coarse quantizer (niter 25, <=256 pts/centroid, seed 1234) and, for IVF_PQ,
 * M residual sub-quantizer codebooks.  FLAT / HNSW: no-op. */
int kb2_index_train(kb2_index_t h, const float* x, int64_t n);
/* IndexNode::Add (index_node.h:140-146, ivf.cc:809-844, flat.cc Add).  ids==NULL => sequential
 * labels continuing from Count(). */
int kb2_index_add(kb2_index_t h, const float* x, int64_t n, const int64_t* ids);

/* Typed variants: element type of x / queries.  The reference registers FLAT / IVF_* for fp16, bf16 and int8 through a
 * wrapper that converts the dataset and every query batch to fp32 (index_factory.h:95-103,
 * index_node_data_mock_wrapper.cc:24-60); these entry points do that conversion on the device.  Distances are fp32. */
enum { KB2_DTYPE_F32 = 0, KB2_DTYPE_F16 = 1, KB2_DTYPE_BF16 = 2, KB2_DTYPE_INT8 = 3 };
int kb2_index_train_typed(kb2_index_t h, const void* x, int dtype, int64_t n);
int kb2_index_add_typed(kb2_index_t h, const void* x, int dtype, int64_t n, const int64_t* ids);
int kb2_index_search_typed(kb2_index_t h, const void* queries, int dtype, int64_t nq, int k, const char* json,
                           const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist);

/* IndexNode::Search (index_node.h:164-166; ivf.cc:887-1168; flat.cc:75-152;
 * faiss_hnsw.cc:1344-1527).  json: search keys k is passed explicitly; nprobe, ef,
 * refine_k (ivf_config.h:33-45,97-128; base_hnsw_config.h:40-71).
 * out_ids[nq*k], out_dist[nq*k] are caller-allocated (like BruteForce::SearchWithBuf,
 * include/knowhere/comp/brute_force.h:33-36).
 * k range: FLAT 1..16384; IVF_FLAT / IVF_PQ k (x refine_k with refine) <= 16384; HNSW 1..16384 when the
 * exact branch runs (k >= n/2 or an almost fully filtered bitset), otherwise as far as the beam (ef) fits; sharded
 * searches world * k <= 8192 and k (x refine_k) <= 1024.  Beyond: KB2_INVALID_ARGS.  IVF nprobe (Search, RangeSearch):
 * above 65536 KB2_OUT_OF_RANGE_IN_JSON, else clamped to [1, nlist]; a sharded Search takes at most 1008 probes
 * (KB2_OUT_OF_RANGE_IN_JSON beyond).  Same for kb2_index_search_typed. */
int kb2_index_search(kb2_index_t h, const float* queries, int64_t nq, int k, const char* json,
                     const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist);

/* IndexNode::RangeSearch (index_node.h:253-255; flat.cc:154-234; ivf.cc:1229-1500;
 * include/knowhere/range_util.h:23-26): L2 keeps radius > d >= range_filter,
 * IP keeps radius < d <= range_filter.  has_range_filter=0 => one-sided.
 * Outputs are malloc'ed HOST arrays owned by the caller (free with kb2_free):
 * lims[nq+1], ids[lims[nq]], dist[lims[nq]], each query's hits sorted best-first. */
int kb2_index_range_search(kb2_index_t h, const float* queries, int64_t nq, float radius,
                           float range_filter, int has_range_filter, const char* json,
                           const uint8_t* bitset, int64_t bitset_nbits, int64_t** out_lims,
                           int64_t** out_ids, float** out_dist);
void kb2_free(void* p);

/* IndexNode::Count / Dim / Size / HasRawData / GetVectorByIds (index_node.h:270-279,329-395) */
int64_t kb2_index_count(kb2_index_t h);
int kb2_index_dim(kb2_index_t h);
int64_t kb2_index_size_bytes(kb2_index_t h);
int kb2_index_is_trained(kb2_index_t h);
int kb2_index_has_raw_data(kb2_index_t h);
int kb2_index_get_vector_by_ids(kb2_index_t h, const int64_t* ids, int64_t n, float* out);

/* ---- importing an index built elsewhere (a Milvus/faiss CPU-built index) ---------------
 * These replace the Deserialize path for already-parsed faiss structures
 * (reference: K/impl/index_read.cpp IwFl/IwPQ/IHNf readers; SURVEY §8f rank 2) and are what
 * the parity tests use so that GPU and CPU search the *same* trained index.
 * IVF: centroids[nlist*dim]; pq_centroids[M*ksub*dsub] (NULL for IVF_FLAT).  Then one
 * kb2_ivf_import_list per inverted list (codes: list_size*code_size bytes where code_size is
 * M for IVF_PQ nbits=8, dim*4 for IVF_FLAT), then kb2_ivf_import_finish.  raw (optional,
 * n*dim fp32 in label order 0..n-1) enables refine. */
int kb2_ivf_import_begin(kb2_index_t h, int64_t nlist, const float* centroids, const float* pq_centroids);
int kb2_ivf_import_list(kb2_index_t h, int64_t list_no, int64_t list_size, const int64_t* ids,
                        const uint8_t* codes);
int kb2_ivf_import_finish(kb2_index_t h, const float* raw, int64_t n_raw);
/* export (for serialisation to the faiss wire format by the caller / for oracle checks) */
int64_t kb2_ivf_nlist(kb2_index_t h);
int64_t kb2_ivf_list_size(kb2_index_t h, int64_t list_no);
int kb2_ivf_export_centroids(kb2_index_t h, float* centroids, float* pq_centroids);
int kb2_ivf_export_list(kb2_index_t h, int64_t list_no, int64_t* ids, uint8_t* codes);

/* HNSW graph import/export in the reference's own layout (K/impl/HNSW.h: levels[n] (level+1 per
 * node), offsets[n+1], neighbors[offsets[n]] int32 with -1 padding, cum_nneighbor_per_level,
 * entry_point, max_level; K/impl/HNSW.cpp:53-89,202-225).  vectors: n*dim fp32. */
int kb2_hnsw_import(kb2_index_t h, int64_t n, const float* vectors, const int32_t* levels,
                    const int64_t* offsets, const int32_t* neighbors, const int32_t* cum_nneighbor,
                    int n_cum, int32_t entry_point, int32_t max_level);
int kb2_hnsw_export_meta(kb2_index_t h, int64_t* out5 /* n, entry_point, max_level, n_links, n_cum */);
int kb2_hnsw_export(kb2_index_t h, int32_t* levels, int64_t* offsets, int32_t* neighbors, int32_t* cum);
/* per-search statistics of the last kb2_index_search on an HNSW handle
 * (reference HNSWStats: K/impl/HnswSearcher.h:284-288): out2 = {ndis, nhops} summed over queries */
int kb2_hnsw_last_stats(kb2_index_t h, int64_t* out2);

/* ---- Serialize / Deserialize (index_node.h:337-367; BinarySet payload) -------------------
 * Self-describing little-endian blob ("KB2I" container); *out is malloc'ed (kb2_free). */
int kb2_index_serialize(kb2_index_t h, uint8_t** out, size_t* out_size);
int kb2_index_deserialize(const uint8_t* blob, size_t size, int device, kb2_index_t* out);

/* ---- the reference's wire format: faiss fourcc streams, i.e. the payload Knowhere stores in a BinarySet under the
 * index type name (flat.cc:323-343, ivf.cc:1717-1741, faiss_hnsw.cc:188-217; K/impl/index_write.cpp:523-560,716-745,
 * 776-822, K/impl/index_read.cpp).  Supported: "IxF2"/"IxFI"/"IxF9" (FLAT), "IwFl" (IVF_FLAT), "IwPQ" and "IxRF" over it
 * (IVF_PQ, + flat fp32 refine store), "IHNf"/"IHN9" (HNSW over flat storage).  with_norm = 1 when the inverted lists
 * carry per-row norms (the reference's IO_FLAG_WITH_NORM).  A CPU-built Knowhere index loads straight onto the GPU and
 * a GPU-built index can be served by the reference's CPU nodes.  kb2_faiss_describe parses on the host only (no device
 * needed) and returns a one-line JSON description. */
int kb2_faiss_describe(const uint8_t* blob, size_t size, int with_norm, char* json_out, size_t cap);
/* host-only: parse the stream and write it again with this library's writer (out: malloc'ed, kb2_free) */
int kb2_faiss_rewrite(const uint8_t* blob, size_t size, int with_norm, uint8_t** out, size_t* out_size);
int kb2_index_deserialize_faiss(const uint8_t* blob, size_t size, int with_norm, int device, kb2_index_t* out);
int kb2_index_serialize_faiss(kb2_index_t h, uint8_t** out, size_t* out_size);
/* IndexNode::DeserializeFromFile / GetIndexMeta (include/knowhere/index/index_node.h:329-395): the file may hold a
 * faiss stream or this library's "KB2I" container; the meta is a JSON object (type, dim, rows, metric_type, ...) */
int kb2_index_deserialize_from_file(const char* path, int device, kb2_index_t* out);
int kb2_index_get_meta(kb2_index_t h, char* json_out, size_t cap);

/* ---- index-less exact search: knowhere::BruteForce (include/knowhere/comp/brute_force.h:26-69;
 * src/common/comp/brute_force.cc:260-392,588-710).  k: 1..16384 (KB2_INVALID_ARGS beyond). */
int kb2_bruteforce_search(const float* base, int64_t nb, int dim, int metric, const float* queries,
                          int64_t nq, int k, const uint8_t* bitset, int64_t bitset_nbits,
                          int64_t* out_ids, float* out_dist, int device, void* cuda_stream);
int kb2_bruteforce_range_search(const float* base, int64_t nb, int dim, int metric, const float* queries,
                                int64_t nq, float radius, float range_filter, int has_range_filter,
                                const uint8_t* bitset, int64_t bitset_nbits, int64_t** out_lims,
                                int64_t** out_ids, float** out_dist, int device, void* cuda_stream);

/* ---- sparse float vectors: SPARSE_INVERTED_INDEX / SPARSE_WAND (src/index/sparse/sparse_index_node.cc) and
 * BruteForce::SearchSparse (src/common/comp/brute_force.cc:1227-1340).  DESIGN §4.13.
 * A row set is CSR: indptr int64[n + 1] (indptr[0] = 0, non-decreasing), indices uint32[indptr[n]] strictly ascending
 * within a row, values float32[indptr[n]] finite and >= 0; each array host or device.  Anything else is
 * KB2_INVALID_ARGS before any kernel indexes by the data.  Scores, evaluated in fp32 in this order:
 *   IP:   s(q, r) = sum over the kept query entries (t, w) that row r holds (value v), in query order, of w * v
 *   BM25: the same sum of ((w * (k1 + 1)) * v) / ((v + k1 * (1 - b)) + ((k1 * b) / max(avgdl, 1)) * L_r), L_r = the sum
 *         of row r's values (scorer.h:81-104; avgdl of the search keys)
 * Candidates are the rows with s > 0 the bitset keeps; results are ordered by s descending, ties by ascending row; row ids
 * are positions in add order.  Missing entries: id -1, distance -FLT_MAX (the reference pads with NaN). */
/* IndexNode::Add on a sparse index (sparse_index_node.cc Train + Add): appends n rows; may be called more than once and
 * gives the same index as one call with the concatenated rows.  No custom ids. */
int kb2_index_add_sparse(kb2_index_t h, const int64_t* indptr, const uint32_t* indices, const float* values, int64_t n);
/* IndexNode::Search on a sparse index (sparse_index_node.cc:767-792, inverted_index.h:151-190): the exact top-k, k 1..16384.
 * Search keys: drop_ratio_search in [0, 1) (else KB2_OUT_OF_RANGE_IN_JSON) keeps a query entry when its value is >= the
 * value at position (size_t)(float(ratio) * float(nnz_q)) of the query's values in ascending order (0 when that position
 * is 0); entries whose index no stored row has are dropped too.  BM25: bm25_avgdl is required (KB2_INVALID_ARGS); bm25_k1
 * and bm25_b, if given, must equal the build values (KB2_INVALID_VALUE_IN_JSON).  search_algo, dim_max_score_ratio,
 * refine_factor and bulk_query_nnz_threshold are accepted without effect.  out_ids / out_dist [nq][k], both host or
 * both device.  kb2_index_last_search_counters: [3] postings scored, [2] their bytes (8 each). */
int kb2_index_search_sparse(kb2_index_t h, const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values,
                            int64_t nq, int k, const char* json, const uint8_t* bitset, int64_t bitset_nbits,
                            int64_t* out_ids, float* out_dist);
/* IndexNode::RangeSearch on a sparse index: the hits radius < s <= range_filter (has_range_filter = 0: radius < s) among the
 * candidates, each query's best first, ties by row; same keys as kb2_index_search_sparse and the outputs of
 * kb2_index_range_search. */
int kb2_index_range_search_sparse(kb2_index_t h, const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values,
                                  int64_t nq, float radius, float range_filter, int has_range_filter, const char* json,
                                  const uint8_t* bitset, int64_t bitset_nbits, int64_t** out_lims, int64_t** out_ids,
                                  float** out_dist);
/* BruteForce::SearchSparse (brute_force.cc:1227-1340): nb base rows against nq queries, metric KB2_METRIC_IP or
 * KB2_METRIC_BM25 (json: bm25_k1, bm25_b and bm25_avgdl, as for the index), k 1..16384.  Every query entry is kept (no
 * drop_ratio_search), so the result equals a sparse index's over the same rows at drop_ratio_search 0, bit for bit. */
int kb2_bruteforce_search_sparse(const int64_t* base_indptr, const uint32_t* base_indices, const float* base_values,
                                 int64_t nb, const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values,
                                 int64_t nq, int metric, int k, const char* json, const uint8_t* bitset,
                                 int64_t bitset_nbits, int64_t* out_ids, float* out_dist, int device);

/* ---- emb-list (multi-vector) exact search: knowhere::BruteForce::Search with a MAX_SIM_* metric and EMB_LIST_OFFSET on
 * both datasets (src/common/comp/brute_force.cc:258-300,424-584,626-665; include/knowhere/emb_list_utils.h).
 * Document i is base rows [base_lims[i], base_lims[i+1]), query list j is query rows [query_lims[j], query_lims[j+1]);
 * rows are dim fp32.  Offsets (n_docs + 1 and n_lists + 1 entries, host or device) start at 0 and do not decrease.
 *   score(Q, D) = sum over q in Q of max over x in D of <q, x>      KB2_METRIC_MAX_SIM_IP; _COSINE: unit q and x / |x|
 *   score(Q, D) = sum over q in Q of min over x in D of |q - x|^2   KB2_METRIC_MAX_SIM_L2 (smaller is better)
 * Result [n_lists][k]: document ids best first, ties by ascending id; out_dist is the score itself (not negated).
 * Bit i of the bitset filters out document i; a bitset must cover n_docs bits.  An empty document is never returned.
 * Missing entries have id -1 and distance FLT_MIN (MAX_SIM_IP / _COSINE: std::numeric_limits<float>::min(), as the
 * reference pads, brute_force.cc:566-581) or FLT_MAX (MAX_SIM_L2).  An empty query list gets a whole row of that padding
 * (the reference leaves such a row as allocated, brute_force.cc:653-655).  k: 1..16384.  Malformed offsets or sizes:
 * KB2_INVALID_ARGS; any other metric (MAX_SIM_HAMMING / _JACCARD: no binary vectors here): KB2_INVALID_METRIC_TYPE.
 * out_stats (nullable) int64[3]: query lists, candidate slots re-ranked exactly, lists scored exactly over every document
 * (lists the filter could not certify, or every list when dim % 4 != 0).  DESIGN §4.10. */
int kb2_bruteforce_search_emb_list(const float* base, const int64_t* base_lims, int64_t n_docs, int dim, int metric,
                                   const float* queries, const int64_t* query_lims, int64_t n_lists, int k,
                                   const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist,
                                   int64_t* out_stats, int device, void* cuda_stream);

/* ---- emb-list (multi-vector) search on an index: the reference's TokenANN strategy on HNSW and IVF_FLAT
 * (src/index/emb_list/emb_list_strategy_token_ann.cc:51-175, emb_list_strategy.cc:45-117, index_node.cc:275-324,453-657).
 * kb2_index_set_emb_list attaches document offsets to an HNSW or IVF_FLAT handle whose rows are added or imported:
 * document i is rows [lims[i], lims[i+1]); lims (n_docs + 1 entries, host or device) start at 0, do not decrease and
 * end at kb2_index_count (else KB2_INVALID_ARGS).  metric pairs with the index metric: MAX_SIM_L2 with L2, MAX_SIM_IP
 * with IP, MAX_SIM_COSINE with COSINE; any other pairing, and FLAT / IVF_PQ, give KB2_INVALID_METRIC_TYPE.  A sharded
 * handle or one with custom ids: KB2_NOT_IMPLEMENTED.  Once attached, kb2_index_search / _range_search return
 * KB2_EMB_LIST_INNER_ERROR, and kb2_index_add / _train, kb2_hnsw_import and kb2_ivf_import_* KB2_NOT_IMPLEMENTED; the
 * "KB2I" blob keeps the offsets.
 * kb2_index_emb_list_offsets: *n_docs, and the offsets into lims (n_docs + 1 entries) when lims is not NULL
 * (KB2_INVALID_ARGS on a handle without emb-lists).
 * kb2_index_search_emb_list: query list j is query rows [query_lims[j], query_lims[j+1]).  json: retrieval_ann_ratio
 * (default 3; <= 0 is KB2_EMB_LIST_INNER_ERROR) and the base search keys (ef, nprobe, disable_fallback_brute_force).
 * Every query token is searched on the base index for vec_topk = min(max(int(k * ratio), 1), rows) rows (HNSW: ef >= k,
 * the list-level k, and the beam is max(ef, vec_topk)); the distinct documents of a list's hits are its candidates, and
 * their exact MaxSim scores (bit-identical to kb2_bruteforce_search_emb_list's) give the k best.  vec_topk is bounded
 * by the base search's limits, whose error names them.  Bit i of the bitset filters out document i (n_docs bits at
 * least).  Result [n_lists][k]: documents best first, ties by ascending id; padding id -1 with -FLT_MAX (MAX_SIM_IP /
 * _COSINE) or FLT_MAX (MAX_SIM_L2), a whole row of it for an empty query list.  k: 1..16384.  out_stats (nullable)
 * int64[3]: query lists, (list, document) candidates re-ranked, token x row distances computed.  DESIGN §4.11. */
int kb2_index_set_emb_list(kb2_index_t h, const int64_t* lims, int64_t n_docs, int metric);
int kb2_index_emb_list_offsets(kb2_index_t h, int64_t* n_docs, int64_t* lims);
int kb2_index_search_emb_list(kb2_index_t h, const float* queries, const int64_t* query_lims, int64_t n_lists, int k,
                              const char* json, const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids,
                              float* out_dist, int64_t* out_stats);
/* ---- the MUVERA strategy (src/index/emb_list/emb_list_strategy_muvera.cc; DESIGN §4.11): an HNSW or IVF_FLAT handle
 * created with "emb_list_strategy": "muvera" (default, or an empty string: "tokenann"; "lemur": KB2_NOT_IMPLEMENTED; any
 * other string: KB2_INVALID_ARGS; other index types do not read these keys and refuse kb2_index_set_emb_list), "muvera_num_projections" P (1..7, default 4), "muvera_num_repeats" R (1..32, default 7) and
 * "muvera_seed" S (int32, default 42; out of range: KB2_OUT_OF_RANGE_IN_JSON).  With token dimension d, B = 2^P buckets
 * and E = R * B * d encoded dimensions.  On such a handle kb2_index_add keeps the token rows (raw, also under COSINE),
 * kb2_index_train does nothing and kb2_index_count is the token-row count; kb2_index_search / _range_search return
 * KB2_EMB_LIST_INNER_ERROR and kb2_hnsw_* / kb2_ivf_* KB2_NOT_IMPLEMENTED.  kb2_index_set_emb_list (same checks as
 * above) encodes every document into its Fixed Dimensional Encoding (per repeat and bucket the mean of its tokens in
 * the bucket) and builds the base index of the handle's type over the n_docs encoded rows (IVF_FLAT: its k-means and
 * nlist cap; HNSW: its build); a second kb2_index_set_emb_list on such a handle is KB2_NOT_IMPLEMENTED.  A base that cannot serve E fails here or at search with its own error (limits:
 * kb2_emb_list_index.cuh).  kb2_index_search_emb_list encodes each query list (the sum of its tokens per bucket),
 * searches the base for ann_k documents and, with "emb_list_rerank" true (default), re-ranks them by exact MaxSim as
 * above: ann_k = min(max(int(k * ratio), 1), n_docs); the bitset filters documents of the base directly; a list gets
 * the k best of its candidates, empty documents skipped, padded as above.  With emb_list_rerank false: ann_k =
 * min(k, n_docs), the base's ids and distances as they are, padded with -1 and -inf (MAX_SIM_IP / _COSINE) or +inf.
 * The "KB2I" blob holds the base, P, R, S, d, the offsets and the token rows; the faiss stream: KB2_NOT_IMPLEMENTED.
 * GetIndexMeta adds emb_list_strategy, muvera_num_projections, muvera_num_repeats, muvera_seed and muvera_encoded_dim.
 *
 * device ms of the stages of the last kb2_index_search_emb_list on this handle (with kb2_index_enable_kernel_timing):
 * out4 = stage 1 (base search; MUVERA: encode + base search), candidates, re-rank, select + emit */
int kb2_index_emb_list_stage_ms(kb2_index_t h, float* out4);

/* ---- multi-GPU: one process per GPU, inverted lists sharded (kb2_index_set_shard), collectives over NCCL/NVLink
 * INSIDE the library (SURVEY §8e; the reference has no multi-GPU path: one index per device,
 * src/common/cuvs/integration/cuvs_knowhere_index.cuh:415-460).  Bootstrap as in NCCL: rank 0 obtains a 128-byte id,
 * the host application distributes it (its own RPC; torch.distributed in the tests), every rank creates its
 * communicator on its device.  After kb2_index_set_comm, kb2_index_search on a sharded IVF index is a COLLECTIVE call:
 * every rank passes the same query batch and receives the same global top-k.  Per call: the coarse quantizer runs on
 * 1/world of the batch per rank + one all-gather of the probe lists; (tensor-core IVF_PQ engine) phase-A bounds are
 * computed by the rank owning each query's nearest list + one min all-reduce; every rank scans its own lists; ONE
 * all-gather of the per-shard top-k candidates + the merge kernel.  NCCL is resolved with dlopen("libnccl.so.2"). */
int kb2_comm_unique_id(uint8_t* out128);
int kb2_comm_create(const uint8_t* id128, int rank, int world, int device, kb2_comm_t* out);
void kb2_comm_destroy(kb2_comm_t c);
/* every rank contributes `bytes` device bytes; recv holds world*bytes, rank-major (exposed for tests / host glue) */
int kb2_comm_all_gather(kb2_comm_t c, const void* send, void* recv, size_t bytes, void* cuda_stream);
/* attach (or detach with NULL) a communicator; rank/world/device must equal the handle's shard settings.  The
 * communicator is not owned by the index and must outlive it. */
int kb2_index_set_comm(kb2_index_t h, kb2_comm_t c);

/* ---- multi-GPU candidate merge (the kernel that consumes the NCCL all-gather, SURVEY §8e) ---
 * in_ids/in_dist: [world][nq][k] gathered per-shard results (device or host);
 * out: [nq][k] global top-k, same ordering rules as search. */
int kb2_merge_topk(int metric, int world, int64_t nq, int k, const int64_t* in_ids, const float* in_dist,
                   int64_t* out_ids, float* out_dist, int device, void* cuda_stream);

/* ---- introspection used by bench.py for the roofline figures --------------------------- */
/* fills out[0..7] with counters of the last search on this handle:
 * [0] kernels launched, [1] codes (rows) scanned, [2] algorithmic code bytes scanned,
 * [3] (query,list) pairs, [4] H2D bytes, [5] D2H bytes, [6] IVF_PQ tensor-core engine: codes re-evaluated exactly (survivors of
 * the bf16 filter), [7] queries redone by the LUT kernel (no bound / survivor-buffer overflow) */
int kb2_index_last_search_counters(kb2_index_t h, int64_t* out8);
/* device time in milliseconds of the dominant scan kernel of the last search, measured with
 * CUDA events on the handle's stream (valid only after kb2_index_enable_kernel_timing(h,1)) */
int kb2_index_enable_kernel_timing(kb2_index_t h, int on);
int kb2_index_last_kernel_ms(kb2_index_t h, float* out_ms);
/* out4: [0] device ms of the whole list-scan stage of the last search, [1] device ms of its dominant kernel
 * (== kb2_index_last_kernel_ms), [2] engine that served it: 0 = query-major scan kernels, 1 = list-major
 * tensor-core engine (IVF_PQ m=16 d=128 with large batches; kb2_ivfpq_tc.cuh), 2 = large-k path, 3 = HNSW beam
 * search with one query per CTA (max(ef, k) too large for the four-queries-per-CTA kernels), 4 = GPU_CAGRA, 5 = sparse tile
 * scoring (a sparse search with k + 16 > 1024 reports 2), [3] device ms of the collectives
 * (+ merge kernel) of a sharded search with a communicator */
int kb2_index_last_stage_info(kb2_index_t h, float* out4);

/* validation hook: writes the full key matrix [nq][round_up(nb,4)] of the dense contraction
 * (|q|^2+|x|^2-2qx for L2, -qx for IP) computed by the fp32 CUDA-core kernel (use_tc=0) or by the
 * wgmma tensor-core kernel (use_tc=1).  Device pointers only.  Used by tests to hold the tensor-core
 * path to the fp32 one (the reference computes these distances with src/simd fvec_L2sqr_ny). */
int kb2_debug_gemm_keys(const float* q, int64_t nq, const float* x, int64_t nb, int dim, int metric, int use_tc,
                        float* out_keys, int device);

/* validation hook: the k-means of the IVF build (the coarse quantizer and every PQ sub-quantizer are trained by it) over
 * the n rows x (device, n x dim fp32): k centroids, metric KB2_METRIC_L2 or KB2_METRIC_IP, niter Lloyd iterations from a
 * std::mt19937_64 seeded with seed (IVF build: niter 25, seed 1234).  niter = 0 returns the initial centroids.
 * out_centroids: device, k x dim fp32.  n < k: KB2_INVALID_ARGS.  Used by tests to hold each Lloyd step to a numpy
 * model (DESIGN §4.8). */
int kb2_debug_kmeans(const float* x, int64_t n, int dim, int k, int metric, int niter, uint64_t seed,
                     float* out_centroids, int device);

/* validation hook: the MUVERA encoder (DESIGN §4.11) over n_items items, item i being the rows [lims[i], lims[i+1]) of x
 * (n x dim fp32; x and lims host or device).  out_projections (nullable, host or device, R x P x dim fp32): the
 * projections drawn from num_projections P, num_repeats R and seed; out_fde (nullable, host or device, n_items x E fp32,
 * E = R * 2^P * dim): the encodings, mean != 0 as documents (kb2_index_set_emb_list), 0 as query lists.  Used by tests to
 * hold the projections to the C++ standard library and the encodings to a numpy model. */
int kb2_debug_muvera_encode(const float* x, const int64_t* lims, int64_t n_items, int dim, int num_projections,
                            int num_repeats, int seed, int mean, float* out_projections, float* out_fde, int device);

/* validation hook: step 1 of the GPU_CAGRA build alone (DESIGN §4.12) over the n rows x (device, n x dim fp32), with
 * the build keys of json (intermediate_graph_degree, build_algo, nn_descent_niter; errors as kb2_index_create).  metric:
 * KB2_METRIC_L2 or KB2_METRIC_IP.  m = min(intermediate_graph_degree, n - 1); out_ids (device, n x m int32) receives
 * G0, best first, and out_keys (device, n x m) their keys (squared L2, or minus the inner product).  *out_iters: the
 * NN-descent iterations run (0 for the exact graph); out_updates (host, up to updates_cap entries): updates(t) of each;
 * *out_ms: device ms of the step.  out_iters, out_updates and out_ms may be NULL.  Used by tests to hold the device
 * graph to the numpy model and to measure its recall. */
int kb2_debug_cagra_knn_graph(const float* x, int64_t n, int dim, int metric, const char* json, int32_t* out_ids,
                              float* out_keys, int* out_iters, int64_t* out_updates, int updates_cap, float* out_ms,
                              int device);

#ifdef __cplusplus
}
#endif
#endif /* KNOWHERE_B200_H */
