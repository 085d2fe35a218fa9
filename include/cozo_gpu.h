/*
 * cozo_gpu.h — C ABI of libcozo_gpu.so, the H100 (sm_90a) implementation of
 * CozoDB's HNSW k-NN search and FixedRule graph algorithms.
 *
 * This is the drop-in boundary: every entry point below is what the reference's
 * Rust host code would bind over `extern "C"` (see INTEGRATION.md for the Rust
 * side).  Plain pointers and sizes only.  Citations are file:line under
 * /root/reference/cozo-core/src/.
 *
 * Conventions
 *   - return 0 on success, a negative COZO_GPU_E* code on failure; the message
 *     is available from cozo_gpu_last_error() (thread-local).
 *   - pointers are caller-owned HOST memory unless the parameter / function name
 *     says `_dev` (device memory on the current device).
 *   - ids are dense u32.  HNSW ids are assigned by the host (Rust) side, which keeps the
 *     id <-> (Tuple key, field, sub-index) table (CompoundKey, hnsw.rs:55); graph node ids
 *     are assigned by the host too (cozo_gpu_graph_stage) or on the device from the node
 *     keys' memcmp encodings (cozo_gpu_graph_stage_keys), fixed_rule/mod.rs:144-179.
 *   - there is NO CPU fallback: without a usable sm_90 device init fails.
 *   - search calls are re-entrant per handle: each call takes its own stream and
 *     a workspace from a bounded pool.  Graph algorithm calls are thread-safe per
 *     handle too (the staged graph is read-only, every call owns its buffers) but
 *     run on the default stream, i.e. concurrent calls serialise on the device.
 *     stage / free / build / insert / insert_at / update / remove / compact are not concurrent with
 *     any other call on the same handle.
 *   - `poison` parameters point at a 32-bit flag mirroring the AtomicBool inside
 *     Poison (runtime/db.rs:1926-1942; INTEGRATION.md shows the mirror); it is
 *     polled between kernel launches and makes the call return COZO_GPU_EKILLED,
 *     mirroring `poison.check()?`.
 */
#ifndef COZO_GPU_H
#define COZO_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COZO_GPU_OK 0
#define COZO_GPU_EINVAL (-1)   /* bad argument (dimension mismatch, k==0, ...) */
#define COZO_GPU_ECUDA (-2)    /* CUDA runtime / driver error                  */
#define COZO_GPU_ENODEV (-3)   /* no sm_90 device / extension unusable         */
#define COZO_GPU_ENOMEM (-4)   /* allocation failed                            */
#define COZO_GPU_EKILLED (-5)  /* poison flag was set (runtime/db.rs:1933-1941) */
#define COZO_GPU_EUNSUP (-6)   /* outside the supported envelope (e.g. maintenance of an F64 index) */

#define COZO_GPU_NONE 0xFFFFFFFFu /* padding id in result arrays */
#define COZO_GPU_MAX_PEERS 16     /* destinations of the fused search + exchange */

/* HnswDistance — parse/sys.rs:94-98; formulas hnsw.rs:66-109 */
#define COZO_GPU_L2 0     /* sum (a-b)^2, squared, no sqrt      */
#define COZO_GPU_COSINE 1 /* 1 - a.b / sqrt(|a|^2 |b|^2)       */
#define COZO_GPU_IP 2     /* 1 - a.b                            */

/* ---- lifecycle ---------------------------------------------------------- */
/* Binds the calling process to `device` (ordinal) and verifies it is sm_90. */
int cozo_gpu_init(int device);
void cozo_gpu_shutdown(void);
const char* cozo_gpu_last_error(void);
int cozo_gpu_device_count(void);
/* tuning knobs ("hnsw.mode", "hnsw.warps_per_cta", "hnsw.stages", ...) */
int cozo_gpu_set_option(const char* name, int64_t value);
int64_t cozo_gpu_get_option(const char* name);

/* ---- HNSW --------------------------------------------------------------- */
typedef struct cozo_gpu_hnsw cozo_gpu_hnsw_t;

/* One layer of the index after the reading rules of hnsw_get_neighbours
 * (hnsw.rs:588-629) were applied by the host: rows whose to-key equals the
 * from-key (self-loop, sibling vectors of one row; hnsw.rs:609) and rows with
 * ignore_link (hnsw.rs:618-620) removed.  levels[L] is reference layer -L. */
typedef struct {
  uint32_t n_nodes;         /* rows in this layer                                   */
  const uint32_t* node_ids; /* [n_nodes] ascending dense ids; NULL on layer 0 (all) */
  const uint64_t* row_ptr;  /* [n_nodes+1]                                          */
  const uint32_t* col_idx;  /* [row_ptr[n_nodes]] dense ids, key order within a row */
} CozoGpuHnswLevel;

/* Parameter block of staging; the manifest fields are HnswIndexManifest
 * (hnsw.rs:27-43) as derived in runtime/relation.rs:1136-1151. */
typedef struct {
  uint32_t n_vectors;
  uint32_t dim;           /* vec_dim                                   */
  int32_t metric;         /* COZO_GPU_L2 / COSINE / IP                 */
  uint32_t n_levels;      /* >= 1; top layer = -(n_levels-1)           */
  const CozoGpuHnswLevel* levels;
  const void* vectors;    /* row-major [n_vectors x dim], f32 or f64 per vec_dtype */
  int32_t vectors_on_device; /* 0: host pointer, 1: device pointer     */
  uint32_t entry_point;   /* fr part of the first index row in key order
                             (hnsw.rs:891-899); COZO_GPU_NONE = canary only = empty index */
  uint32_t m_max0;        /* 2*m, degree bound on layer 0              */
  uint32_t m_max;         /* m, degree bound above                     */
  int32_t vec_dtype;      /* VecElementType (data/relation.rs:108): 0 = F32, 1 = F64.  An F64 index keeps f64
                             payloads and is searched with cozo_gpu_hnsw_search_f64 only */
} CozoGpuHnswStageDesc;

typedef struct {
  uint64_t n_queries;
  uint64_t dist_evals;     /* VectorCache::dist calls (hnsw.rs:573,916)        */
  uint64_t nodes_expanded; /* hnsw_get_neighbours calls (hnsw.rs:566-567)      */
  uint64_t nbr_reads;      /* neighbour ids read = sum of expanded degrees     */
  double kernel_ms;        /* device time of the search kernel (CUDA events)   */
} CozoGpuSearchStats;

/* Builds the HBM-resident copy: padded-CSR adjacency per layer + f32 matrix.  Any dim stages.  Width envelope of
 * the f32 search, build and maintenance calls: any dim whose query (round_up(dim,4)*4 bytes), one row stage of the
 * same size and the ef beam fit the device's shared-memory opt-in (227 KB on an H100: up to about 28 000 elements);
 * beyond it those calls return COZO_GPU_EUNSUP naming dim, ef and the bytes needed.  (Forcing the cooperative search,
 * option "hnsw.mode" = 2, needs a row stage per warp: up to about 11 500 elements.) */
int cozo_gpu_hnsw_stage(cozo_gpu_hnsw_t** out, const CozoGpuHnswStageDesc* desc);
void cozo_gpu_hnsw_free(cozo_gpu_hnsw_t* h);

/* Batched SessionTx::hnsw_knn (hnsw.rs:869-1012) without the base-row fetch,
 * bind_* columns and filter bytecode, which stay on the host:
 *   per query: entry point -> ef=1 search on layers top..-1 -> ef search on
 *   layer 0 -> trim to k -> drop dist > radius -> nearest first.
 * radius < 0 means None.  With a `filter` the host passes k := ef and truncates
 * itself (hnsw.rs:943-947,997-1006).
 * out_ids [B*k] padded with COZO_GPU_NONE, out_dist [B*k] padded with +inf,
 * out_count [B] (nullable), stats nullable.  Widths: see cozo_gpu_hnsw_stage (EUNSUP beyond the envelope). */
int cozo_gpu_hnsw_search(cozo_gpu_hnsw_t* h, const float* queries, uint32_t B, uint32_t k, uint32_t ef,
                         double radius, uint32_t* out_ids, float* out_dist, uint32_t* out_count,
                         CozoGpuSearchStats* stats);

/* Same with every buffer already resident in HBM; asynchronous on `stream`
 * (a cudaStream_t, NULL = legacy default stream).  per_query_stats_dev: nullable
 * u32 [B*4] = {dist_evals, nodes_expanded, nbr_reads, f32 rows fetched}; the last is below dist_evals when
 * the search (of any metric) rejected neighbours from their uint8 code rows alone, and equals it otherwise. */
int cozo_gpu_hnsw_search_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k, uint32_t ef,
                             double radius, uint32_t* out_ids_dev, float* out_dist_dev, uint32_t* out_count_dev,
                             uint32_t* per_query_stats_dev, void* stream);

/* hnsw_knn with a `filter` (hnsw.rs:943-947, 997-1006): the beam is NOT trimmed to k before the filter; rows
 * are dropped where the filter bytecode is false and only then the first k are kept.  The host evaluates the
 * filter once per indexed row (possible whenever the expression does not read the bound distance) and passes
 * the verdicts as a bit mask: bit (id & 31) of word id >> 5 set = row `id` passes; [ceil(n_vectors/32)] words.
 * The trim happens inside the kernel, so only k results per query travel back. */
int cozo_gpu_hnsw_search_filtered(cozo_gpu_hnsw_t* h, const float* queries, uint32_t B, uint32_t k, uint32_t ef,
                                  double radius, const uint32_t* row_mask, uint32_t* out_ids, float* out_dist,
                                  uint32_t* out_count, CozoGpuSearchStats* stats);
int cozo_gpu_hnsw_search_filtered_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k,
                                      uint32_t ef, double radius, const uint32_t* row_mask_dev, uint32_t* out_ids_dev,
                                      float* out_dist_dev, uint32_t* out_count_dev, uint32_t* per_query_stats_dev,
                                      void* stream);

/* hnsw_knn on an F64 index (manifest.dtype == F64): the query is f64 (an F32 query is widened by the caller,
 * hnsw.rs:879-884), distances are computed and returned in f64 (hnsw.rs:73-76, 86-93, 102-107).  row_mask as in
 * cozo_gpu_hnsw_search_filtered, nullable.  F64 indexes are search-only on the device: insert / update / remove
 * answer COZO_GPU_EUNSUP and the host re-stages after a mutation. */
int cozo_gpu_hnsw_search_f64(cozo_gpu_hnsw_t* h, const double* queries, uint32_t B, uint32_t k, uint32_t ef,
                             double radius, const uint32_t* row_mask, uint32_t* out_ids, double* out_dist,
                             uint32_t* out_count, CozoGpuSearchStats* stats);

/* Sharded corpus, fused search + exchange (SURVEY.md §8e): the search kernel stores the top-k of
 * every query straight into the [n_slots][B][k] gather buffers of all `n_dest` destinations at
 * slot `slot` (this rank) — peer GPUs' buffers mapped into this process over NVLink (CUDA IPC /
 * symmetric memory; the pointers are passed as integers) — so the all-gather needs no separate
 * collective.  The caller synchronises the ranks (any cross-GPU barrier) before merging with
 * cozo_gpu_topk_merge_dev.  Padding as in cozo_gpu_hnsw_search. */
int cozo_gpu_hnsw_search_scatter_dev(cozo_gpu_hnsw_t* h, const float* queries_dev, uint32_t B, uint32_t k,
                                     uint32_t ef, double radius, uint32_t n_dest, const uint64_t* dest_ids_ptrs,
                                     const uint64_t* dest_dist_ptrs, uint32_t slot, uint32_t* per_query_stats_dev,
                                     void* stream);

/* Index construction on the device (batched variant of hnsw_put_vector,
 * hnsw.rs:155-375: level law 46-52, ef_construction search 242-256, heuristic
 * selection 470-538, shrink 376-469).  Inserts in id order like
 * create_hnsw_index's bulk insert (runtime/relation.rs:1176-1185). */
typedef struct {
  uint32_t n_vectors;
  uint32_t dim;
  int32_t metric;
  const float* vectors;
  int32_t vectors_on_device;
  int32_t borrow_vectors;       /* 1: keep using the caller's device buffer (must outlive the handle) */
  uint32_t m_neighbours;        /* m; m_max = m, m_max0 = 2m, level_multiplier = 1/ln m */
  uint32_t ef_construction;
  int32_t extend_candidates;    /* hnsw.rs:499-511.  Order-dependent: inserts one node per batch and links its
                                   neighbours one at a time (the reference's sequential semantics); for small indexes */
  int32_t keep_pruned_connections;
  uint64_t level_seed;
  uint32_t max_batch;           /* 0 = default */
} CozoGpuHnswBuildDesc;

/* Widths: the envelope of cozo_gpu_hnsw_stage with ef := ef_construction; insert, insert_at and update check it
 * before any row is appended or moved. */
int cozo_gpu_hnsw_build(cozo_gpu_hnsw_t** out, const CozoGpuHnswBuildDesc* desc);

/* Index maintenance on the device, for an index that was built here or staged from the host.
 * insert = hnsw_put for rows whose keys sort after every indexed key (query/stored.rs:332 ->
 * hnsw.rs:679-727): the vectors get the dense ids [n, n+count) (*first_id = n), levels from the
 * handle's seeded level law; ef_construction 0 / keep_pruned < 0 keep the handle's settings
 * (a staged index has none: pass them).  An EMPTY index (n = 0, staged from the canary row alone)
 * grows in place: its first vector only gets its rows and becomes the entry point (hnsw.rs:360-373).
 * remove = hnsw_remove (hnsw.rs:728-868): the nodes'
 * rows are deleted on every layer together with every edge that points at them; if the entry
 * point goes, the first remaining row in key order takes over (hnsw.rs:828-865). */
int cozo_gpu_hnsw_insert(cozo_gpu_hnsw_t* h, const float* vectors, uint32_t count, int32_t vectors_on_device,
                         uint32_t ef_construction, int32_t keep_pruned_connections, uint32_t* first_id);
/* hnsw_put of new rows at ANY key position (query/stored.rs:332 -> hnsw.rs:679-727).
 * positions[i] = number of ids already in the index (live or removed) whose compound key sorts before
 * new row i; non-decreasing, <= n; rows with equal positions in key order.  Existing id j becomes
 * j + #{i : positions[i] <= j}; new row i gets id positions[i] + i, so dense ids stay in key order.
 * Levels come from the handle's level law, drawn in row order.  out_ids [count] nullable.
 * Arguments and errors as cozo_gpu_hnsw_insert, plus COZO_GPU_EINVAL for positions that decrease
 * or exceed n.  With every position equal to n the call is cozo_gpu_hnsw_insert.  After the new rows
 * are linked, the entry point is the smallest id on the top layer (hnsw.rs:184-199).  Waits for
 * device work already enqueued on the handle (an asynchronous search_dev) before moving rows. */
int cozo_gpu_hnsw_insert_at(cozo_gpu_hnsw_t* h, const uint32_t* positions, const float* vectors, uint32_t count,
                            int32_t vectors_on_device, uint32_t ef_construction,
                            int32_t keep_pruned_connections, uint32_t* out_ids);
int cozo_gpu_hnsw_remove(cozo_gpu_hnsw_t* h, const uint32_t* ids, uint32_t count);
/* Drop every removed id (cozo_gpu_hnsw_remove, or un-indexed by the host) from the handle.
 * Live id j becomes j - #{removed ids < j}, so dense ids stay in key order.
 * old_to_new [n before the call] (nullable): new id, or COZO_GPU_NONE for a removed id.
 * The map is monotone: stored neighbour order, edge distances, the entry-point rule, the top layer
 * and the level law's state are unchanged; the upper-layer rows of removed ids go too.  Allocated
 * capacity is kept for later inserts.  With no removed id nothing moves; with every id removed the
 * index is empty (n = 0, entry COZO_GPU_NONE), as if staged from the canary row alone.  Waits for
 * device work already enqueued on the handle (an asynchronous search_dev) before moving rows.
 * COZO_GPU_EUNSUP for an F64 index; all scratch is allocated before any row moves, so
 * COZO_GPU_ENOMEM leaves the handle as it was.  A borrowed vector buffer is never written. */
int cozo_gpu_hnsw_compact(cozo_gpu_hnsw_t* h, uint32_t* old_to_new);
/* hnsw_put of a changed vector under an existing key (hnsw.rs:175-182: remove, then insert again);
 * vectors [count x dim] host memory, ids distinct.  The node keeps its id and layer.  Removed ids
 * may be revived this way. */
int cozo_gpu_hnsw_update(cozo_gpu_hnsw_t* h, const uint32_t* ids, const float* vectors, uint32_t count,
                         uint32_t ef_construction, int32_t keep_pruned_connections);

/* Read a staged / built index back as per-layer CSR (rows ascending by id). */
int cozo_gpu_hnsw_info(cozo_gpu_hnsw_t* h, uint32_t* n_vectors, uint32_t* dim, uint32_t* n_levels,
                       uint32_t* entry_point);
int cozo_gpu_hnsw_level_size(cozo_gpu_hnsw_t* h, uint32_t level, uint32_t* n_nodes, uint64_t* n_edges);
int cozo_gpu_hnsw_export_level(cozo_gpu_hnsw_t* h, uint32_t level, uint32_t* node_ids, uint64_t* row_ptr,
                               uint32_t* col_idx);
/* write-back support: the stored `dist` of every edge (aligned with export_level's col_idx) and the
 * liveness of every id, i.e. everything the host needs to re-create the rows of `rel:idx`
 * (runtime/relation.rs:1064-1126) from the device copy. */
int cozo_gpu_hnsw_export_level_dist(cozo_gpu_hnsw_t* h, uint32_t level, float* dist);
int cozo_gpu_hnsw_export_live(cozo_gpu_hnsw_t* h, uint8_t* live);
/* device pointer of the staged f32 matrix and its row stride in floats */
const float* cozo_gpu_hnsw_vectors_dev(cozo_gpu_hnsw_t* h, uint32_t* row_stride);

/* Per-shard top-k merge for the sharded corpus (SURVEY.md §8e): input is the
 * all-gathered [n_shards][B][k] (dist,id) lists, local ids are mapped to global
 * ids by adding shard_offsets[s]; output global top-k nearest first. */
int cozo_gpu_topk_merge_dev(const float* dist_dev, const uint32_t* ids_dev, uint32_t n_shards, uint32_t B,
                            uint32_t k, const uint64_t* shard_offsets_dev, uint64_t* out_ids_dev,
                            float* out_dist_dev, void* stream);

/* ---- sharded corpus: one process per GPU, one shard (vectors + graph) per rank -------------
 * SURVEY.md §8b "Multi-GPU" / §8e.  The reference answers a query from ONE index relation
 * (query/ra.rs:1102-1119 -> runtime/hnsw.rs:869-1012); here the corpus is row-partitioned over the
 * ranks, every rank searches its own shard and the per-shard top-k lists are exchanged and merged
 * inside the library: broadcast + per-shard search + all-gather + merge behind one call.
 * The communicator is NCCL's (resolved with dlopen at first use); its 128-byte unique id is created
 * on one rank and handed to the others by any host channel the embedding process has. */
typedef struct cozo_gpu_shards cozo_gpu_shards_t;
#define COZO_GPU_UID_BYTES 128
int cozo_gpu_shards_unique_id(uint8_t* id /* [COZO_GPU_UID_BYTES] */);
/* collective over `world` ranks (each bound to its own device with cozo_gpu_init) */
int cozo_gpu_shards_init(cozo_gpu_shards_t** out, const uint8_t* id, int rank, int world);
void cozo_gpu_shards_free(cozo_gpu_shards_t* s);
/* exchange: 0 = one NCCL all-gather per list, 1 = peer stores fused into the search kernel (CUDA IPC
 * buffers over NVLink; chosen when every rank could map every peer, option "shard.exchange" = 0 forces NCCL) */
int cozo_gpu_shards_info(cozo_gpu_shards_t* s, int* rank, int* world, int* exchange, uint64_t* total_rows);

/* Collective.  Attach this rank's shard — staged with cozo_gpu_hnsw_stage or built with
 * cozo_gpu_hnsw_build — to the communicator.  Shard r owns the global ids
 * [offset_r, offset_r + n_vectors_r) of the row-contiguous partition.  Every rank also learns every
 * shard's vec_dtype: the f32 searches below answer COZO_GPU_EINVAL on every rank of an F64 group,
 * cozo_gpu_hnsw_search_sharded_f64 on every rank of an F32 group, and all of them on a group whose
 * shards mix the two, before any collective. */
int cozo_gpu_hnsw_stage_sharded(cozo_gpu_shards_t* s, cozo_gpu_hnsw_t* local_shard, uint64_t* out_global_offset,
                                uint64_t* out_total_rows);

/* Collective.  Batched hnsw_knn over the whole sharded corpus.  `queries` [B*dim] is host memory read on
 * rank `root` and broadcast (root >= 0), or passed identically by every rank (root = -1).  Results on
 * every rank that passes out buffers: out_ids [B*k] GLOBAL ids padded with UINT64_MAX, out_dist [B*k]
 * padded with +inf, nearest first; out_count [B] nullable; stats (this rank's shard) nullable.
 * The batch is processed in tiles of "shard.tile" queries (default 65536). */
int cozo_gpu_hnsw_search_sharded(cozo_gpu_shards_t* s, const float* queries, uint32_t B, uint32_t k, uint32_t ef,
                                 double radius, int root, uint64_t* out_ids, float* out_dist, uint32_t* out_count,
                                 CozoGpuSearchStats* stats);
/* Same with the (replicated) batch and the outputs already in HBM; asynchronous, ordered after and
 * before `stream`.  per_query_stats_dev nullable u32 [B*4]. */
int cozo_gpu_hnsw_search_sharded_dev(cozo_gpu_shards_t* s, const float* queries_dev, uint32_t B, uint32_t k,
                                     uint32_t ef, double radius, uint64_t* out_ids_dev, float* out_dist_dev,
                                     uint32_t* per_query_stats_dev, void* stream);

/* Collective.  hnsw_knn with a `filter` over the whole sharded corpus: every shard runs the filtered
 * search of cozo_gpu_hnsw_search_filtered (beam, radius, filter, then the first k) and the per-shard
 * lists are merged as above, so k results per query and rank travel through the exchange.
 * row_mask = this rank's verdicts over its LOCAL ids: bit (id & 31) of word id >> 5,
 * [ceil(n_vectors_local/32)] words; NULL only on a rank whose shard is empty.  A NULL mask on a
 * non-empty shard answers COZO_GPU_EINVAL on that rank alone: the caller makes the same call
 * (filtered or not, same B, k, ef, radius, root) on every rank.  Other arguments as
 * cozo_gpu_hnsw_search_sharded. */
int cozo_gpu_hnsw_search_sharded_filtered(cozo_gpu_shards_t* s, const float* queries, uint32_t B, uint32_t k,
                                          uint32_t ef, double radius, int root, const uint32_t* row_mask,
                                          uint64_t* out_ids, float* out_dist, uint32_t* out_count,
                                          CozoGpuSearchStats* stats);
/* Same with the batch, the mask and the outputs in HBM; asynchronous, ordered after and before `stream`. */
int cozo_gpu_hnsw_search_sharded_filtered_dev(cozo_gpu_shards_t* s, const float* queries_dev, uint32_t B, uint32_t k,
                                              uint32_t ef, double radius, const uint32_t* row_mask_dev,
                                              uint64_t* out_ids_dev, float* out_dist_dev,
                                              uint32_t* per_query_stats_dev, void* stream);
/* Collective.  hnsw_knn over a sharded corpus of F64 shards: every shard runs cozo_gpu_hnsw_search_f64
 * (f64 queries, distances computed and returned in f64) and the lists are merged as above.  `queries`
 * [B*dim] f64 is read on rank `root` and broadcast (root >= 0), or passed identically by every rank
 * (root = -1).  row_mask nullable (no filter), otherwise as cozo_gpu_hnsw_search_sharded_filtered.
 * out_ids [B*k] global ids padded with UINT64_MAX, out_dist [B*k] padded with +inf. */
int cozo_gpu_hnsw_search_sharded_f64(cozo_gpu_shards_t* s, const double* queries, uint32_t B, uint32_t k, uint32_t ef,
                                     double radius, int root, const uint32_t* row_mask, uint64_t* out_ids,
                                     double* out_dist, uint32_t* out_count, CozoGpuSearchStats* stats);

/* ---- graphs (FixedRule algorithms) -------------------------------------- */
typedef struct cozo_gpu_graph cozo_gpu_graph_t;

/* Edge list -> CSR exactly as as_directed_graph / as_directed_weighted_graph
 * hand it to GraphBuilder (fixed_rule/mod.rs:136-200, 208-328): n = max id + 1,
 * adjacency sorted by target, parallel edges kept, weights f32 (mod.rs:306).
 * `undirected` mirroring is done by the caller (mod.rs:187-191). */
int cozo_gpu_graph_stage(cozo_gpu_graph_t** out, uint32_t n, uint64_t m, const uint32_t* src,
                         const uint32_t* dst, const float* w_or_null);
void cozo_gpu_graph_free(cozo_gpu_graph_t* g);
/* as_directed_graph / as_directed_weighted_graph (fixed_rule/mod.rs:136-328) from node KEYS.
 * Endpoint 2e is the `from` key of edge e, endpoint 2e+1 its `to` key, as the byte string
 * key_bytes[key_off[i] .. key_off[i+1]) (key_off [2m+1], non-decreasing).  Two keys are the same
 * node iff their byte strings are equal (the host passes memcmp encodings, data/memcmp.rs).
 * Dense ids are assigned in first-appearance order over endpoints 0, 1, 2, ... (mod.rs:164-179);
 * *out_n = number of distinct keys.  undirected != 0 mirrors every edge right after itself
 * (mod.rs:187-191).  Weights and the CSR: exactly as cozo_gpu_graph_stage, so the handle is one
 * every graph call takes.  COZO_GPU_EINVAL for decreasing offsets or a null pointer when m > 0;
 * COZO_GPU_EUNSUP beyond 2^32-2 edges after mirroring (or 2^31-2 edges before it); COZO_GPU_ENOMEM
 * when the device cannot hold the work, with the bytes needed in the message. */
int cozo_gpu_graph_stage_keys(cozo_gpu_graph_t** out, uint64_t m, const uint8_t* key_bytes,
                              const uint64_t* key_off, const float* w_or_null, int32_t undirected,
                              uint32_t* out_n);
/* for every dense id, the endpoint index (2e or 2e+1) where its key first appeared: out_first [n] */
int cozo_gpu_graph_node_endpoints(cozo_gpu_graph_t* g, uint64_t* out_first);
/* dense id of each key (same byte form), COZO_GPU_NONE where the graph has no such node */
int cozo_gpu_graph_lookup_keys(cozo_gpu_graph_t* g, const uint8_t* key_bytes, const uint64_t* key_off,
                               uint32_t count, uint32_t* out_ids);
/* read the staged CSR back (any pointer nullable): out_ptr/in_ptr [n+1] u32 */
int cozo_gpu_graph_export(cozo_gpu_graph_t* g, uint32_t* out_ptr, uint32_t* out_idx, float* out_w,
                          uint32_t* in_ptr, uint32_t* in_idx);

/* graph::page_rank as called from PageRank::run (algos/pagerank.rs:47-50):
 * PageRankConfig::new(max_iter, tol, damping); returns scores [n] f32. */
int cozo_gpu_pagerank(cozo_gpu_graph_t* g, float damping, double tol, uint32_t max_iter, float* out_scores,
                      uint32_t* out_iters, double* out_err, double* out_kernel_ms, const volatile int* poison);

/* dijkstra (shortest_path_dijkstra.rs:274-339) for many sources at once:
 * out_dist [n_src*n] f32 (+inf unreachable), out_pred [n_src*n] u32 (nullable).
 * goals (nullable) only select which targets the host reads back. */
int cozo_gpu_sssp_multi(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, float* out_dist,
                        uint32_t* out_pred, double* out_kernel_ms, const volatile int* poison);

/* ShortestPathDijkstra with a termination relation (shortest_path_dijkstra.rs:70-150, 274-339): for every source,
 * the shortest paths to `goals` only; each search stops once every goal's distance is final, and each chunk of
 * sources is reduced to its goal answers on the device (host memory O(n_src*n_goals + output), never O(n_src*n)).
 * goals [n_goals] distinct and < n (EINVAL otherwise).  Pair i = si * n_goals + gi.
 * out_cost [n_src*n_goals] f32, +inf unreachable.
 * keep_ties == 0: out_path_off [n_src*n_goals + 1] u64, always written: pair i's path is
 *   out_paths[off[i] .. off[i+1]), start..goal, empty when unreachable.  The paths are complete in out_paths only
 *   when off[n_src*n_goals] <= paths_cap (nothing is written past paths_cap); otherwise call again with a larger
 *   buffer.  out_tie_off / out_tie_edges are not used.
 * keep_ties != 0: no paths.  Instead, per source si, the tied-predecessor edges that lead back from its goals:
 *   out_tie_off [n_src + 1] u64, always written; out_tie_edges[2*off[si] .. 2*off[si+1]) holds (v, p) pairs, one per
 *   CSR edge p -> v with fl32(d[p] + w) == d[v], v != source, v a goal with finite cost or the p of such an edge;
 *   no particular order within a source.  Same capacity convention with ties_cap (in pairs).
 * poison polled between source chunks. */
int cozo_gpu_sssp_goals(cozo_gpu_graph_t* g, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                        uint32_t n_goals, int32_t keep_ties, float* out_cost, uint64_t* out_path_off,
                        uint32_t* out_paths, uint64_t paths_cap, uint64_t* out_tie_off, uint32_t* out_tie_edges,
                        uint64_t ties_cap, double* out_kernel_ms, const volatile int* poison);

/* Goal-directed batch of dijkstra calls with ForbiddenEdge / ForbiddenNode sets, the form
 * KShortestPathYen uses (fixed_rule/algos/yen.rs:138,168; shortest_path_dijkstra.rs:188-218,274-339):
 * search i runs from sources[i] to goals[i]; its forbidden nodes are forb_nodes[forb_node_ptr[i] ..
 * forb_node_ptr[i+1]) and its forbidden (src,dst) pairs the same slice of forb_edge_src/dst (both
 * ptr arrays NULL = no sets).  out_cost [n_src] (+inf unreachable), out_len [n_src] (0 unreachable;
 * > max_len = buffer too small), out_paths [n_src*max_len] node ids start..goal. */
int cozo_gpu_sssp_paths(cozo_gpu_graph_t* g, const uint32_t* sources, const uint32_t* goals, uint32_t n_src,
                        const uint32_t* forb_node_ptr, const uint32_t* forb_nodes, const uint32_t* forb_edge_ptr,
                        const uint32_t* forb_edge_src, const uint32_t* forb_edge_dst, uint32_t max_len,
                        float* out_cost, uint32_t* out_len, uint32_t* out_paths, double* out_kernel_ms,
                        const volatile int* poison);

/* ClosenessCentrality / BetweennessCentrality (all_pairs_shortest_path.rs:97-143, 29-95) */
int cozo_gpu_closeness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms, const volatile int* poison);
int cozo_gpu_betweenness(cozo_gpu_graph_t* g, float* out, double* out_kernel_ms, const volatile int* poison);

/* ClusteringCoefficients (fixed_rule/algos/triangles.rs:25-98) over the out-CSR of the MIRRORED
 * edge stream (as_directed_graph(true), triangles.rs:35): per node (cc f64, n_triangles, degree). */
int cozo_gpu_clustering(cozo_gpu_graph_t* g, double* out_cc, uint64_t* out_triangles, uint64_t* out_degree,
                        double* out_kernel_ms, const volatile int* poison);

/* ---- source-sharded graph calls: the graph replicated on every rank, the sources split -----------------------
 * SURVEY.md §8e "replicate graph, partition sources; no exchange until the end".  The shard group of
 * cozo_gpu_shards_init, one process per GPU; every rank makes the same call with the same arguments.  The
 * sources of a call are split into `world` contiguous slices in source order, slice r = [N*r/world,
 * N*(r+1)/world) of the N sources (empty when world > N); rank r searches slice r with the single-GPU code and
 * every rank returns the complete answer.  Each rank polls its own `poison` between source chunks (once when its
 * slice is empty).  Every call, attach included, first all-gathers one status record per rank: its outcome and the
 * call's signature (which call, the attached graph, n_src, n_goals, keep_ties, the row capacity and a hash of the
 * sources and goals).  When the signatures differ — e.g. two calls reached the group in different orders on
 * different ranks — every rank returns COZO_GPU_EINVAL; otherwise, when any rank failed (an argument check, no
 * graph attached, poison, out of memory, ...), every rank returns the code of the first failing rank in rank
 * order.  So no rank is left waiting, and the group stays usable.  Only a NULL `s` is refused on its rank alone.
 * out_kernel_ms = device time of this rank's slice, before the exchange. */

/* Collective.  Registers `g` — staged on every rank from the same edges with cozo_gpu_graph_stage or
 * cozo_gpu_graph_stage_keys — on the group for the calls below.  Every rank all-gathers (n, m, weighted, a
 * checksum computed on the device over the out-CSR and the bits of its weights); if any rank differs, every rank
 * returns COZO_GPU_EINVAL and the group has no graph (on any rank whose attach fails).  The group does not own `g`: it must outlive its use
 * through the group, and a re-staged graph is attached again. */
int cozo_gpu_graph_attach_sharded(cozo_gpu_shards_t* s, cozo_gpu_graph_t* g);
/* Collective.  cozo_gpu_closeness over the attached graph: the per-source f32 values of every slice are
 * all-gathered, so `out` [n] equals cozo_gpu_closeness bit for bit at every world size. */
int cozo_gpu_closeness_sharded(cozo_gpu_shards_t* s, float* out, double* out_kernel_ms, const volatile int* poison);
/* Collective.  cozo_gpu_betweenness over the attached graph: each rank adds its slice's per-source dependencies in
 * source order in f64, the world partial sums are all-gathered and every rank adds them in rank order and rounds
 * to f32 once, so `out` [n] is the same on every rank and from run to run; at world 1 it equals
 * cozo_gpu_betweenness bit for bit, above it only the association of the f64 sum differs.  COZO_GPU_EUNSUP on
 * every rank when any rank met a zero-weight cycle of tied paths. */
int cozo_gpu_betweenness_sharded(cozo_gpu_shards_t* s, float* out, double* out_kernel_ms, const volatile int* poison);
/* Collective.  cozo_gpu_sssp_goals over the attached graph, with the same arguments, outputs and capacity rule:
 * costs, offsets and rows equal the single-GPU call's (tie edges: the same multiset per source, in no particular
 * order within a source).  Costs, offsets and every slice's row count are all-gathered, then each slice's rows
 * are broadcast from its rank into place.  When the total exceeds paths_cap / ties_cap, costs and offsets are
 * written and no row is. */
int cozo_gpu_sssp_goals_sharded(cozo_gpu_shards_t* s, const uint32_t* sources, uint32_t n_src, const uint32_t* goals,
                                uint32_t n_goals, int32_t keep_ties, float* out_cost, uint64_t* out_path_off,
                                uint32_t* out_paths, uint64_t paths_cap, uint64_t* out_tie_off,
                                uint32_t* out_tie_edges, uint64_t ties_cap, double* out_kernel_ms,
                                const volatile int* poison);

#ifdef __cplusplus
}
#endif
#endif /* COZO_GPU_H */
