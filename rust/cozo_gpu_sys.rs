//! cozo_gpu_sys.rs — raw FFI of libcozo_gpu.so (include/cozo_gpu.h), generated from the header by
//! tools in this repository and checked against it in tests/test_abi_cpu.py.
//! Not compiled in the build image (no Rust toolchain); see rust/README.md.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

pub enum CozoGpuHnsw {}
pub enum CozoGpuGraph {}
pub enum CozoGpuShards {}

pub const COZO_GPU_OK: c_int = 0;
pub const COZO_GPU_EINVAL: c_int = -1;
pub const COZO_GPU_ECUDA: c_int = -2;
pub const COZO_GPU_ENODEV: c_int = -3;
pub const COZO_GPU_ENOMEM: c_int = -4;
pub const COZO_GPU_EKILLED: c_int = -5;
pub const COZO_GPU_EUNSUP: c_int = -6;
pub const COZO_GPU_NONE: u32 = 0xFFFF_FFFF;
pub const COZO_GPU_MAX_PEERS: usize = 16;
pub const COZO_GPU_UID_BYTES: usize = 128;
pub const COZO_GPU_L2: i32 = 0;
pub const COZO_GPU_COSINE: i32 = 1;
pub const COZO_GPU_IP: i32 = 2;

#[repr(C)]
pub struct CozoGpuHnswLevel {
    pub n_nodes: u32,
    pub node_ids: *const u32,
    pub row_ptr: *const u64,
    pub col_idx: *const u32,
}

#[repr(C)]
pub struct CozoGpuHnswStageDesc {
    pub n_vectors: u32,
    pub dim: u32,
    pub metric: i32,
    pub n_levels: u32,
    pub levels: *const CozoGpuHnswLevel,
    pub vectors: *const c_void,
    pub vectors_on_device: i32,
    pub entry_point: u32,
    pub m_max0: u32,
    pub m_max: u32,
    pub vec_dtype: i32,
}

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct CozoGpuSearchStats {
    pub n_queries: u64,
    pub dist_evals: u64,
    pub nodes_expanded: u64,
    pub nbr_reads: u64,
    pub kernel_ms: f64,
}

#[repr(C)]
pub struct CozoGpuHnswBuildDesc {
    pub n_vectors: u32,
    pub dim: u32,
    pub metric: i32,
    pub vectors: *const f32,
    pub vectors_on_device: i32,
    pub borrow_vectors: i32,
    pub m_neighbours: u32,
    pub ef_construction: u32,
    pub extend_candidates: i32,
    pub keep_pruned_connections: i32,
    pub level_seed: u64,
    pub max_batch: u32,
}

#[link(name = "cozo_gpu")]
extern "C" {
    pub fn cozo_gpu_init(device: c_int) -> c_int;
    pub fn cozo_gpu_shutdown();
    pub fn cozo_gpu_last_error() -> *const c_char;
    pub fn cozo_gpu_device_count() -> c_int;
    pub fn cozo_gpu_set_option(name: *const c_char, value: i64) -> c_int;
    pub fn cozo_gpu_get_option(name: *const c_char) -> i64;
    pub fn cozo_gpu_hnsw_stage(out: *mut *mut CozoGpuHnsw, desc: *const CozoGpuHnswStageDesc) -> c_int;
    pub fn cozo_gpu_hnsw_free(h: *mut CozoGpuHnsw);
    pub fn cozo_gpu_hnsw_search(h: *mut CozoGpuHnsw, queries: *const f32, B: u32, k: u32, ef: u32, radius: f64, out_ids: *mut u32, out_dist: *mut f32, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_hnsw_search_dev(h: *mut CozoGpuHnsw, queries_dev: *const f32, B: u32, k: u32, ef: u32, radius: f64, out_ids_dev: *mut u32, out_dist_dev: *mut f32, out_count_dev: *mut u32, per_query_stats_dev: *mut u32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_hnsw_search_filtered(h: *mut CozoGpuHnsw, queries: *const f32, B: u32, k: u32, ef: u32, radius: f64, row_mask: *const u32, out_ids: *mut u32, out_dist: *mut f32, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_hnsw_search_filtered_dev(h: *mut CozoGpuHnsw, queries_dev: *const f32, B: u32, k: u32, ef: u32, radius: f64, row_mask_dev: *const u32, out_ids_dev: *mut u32, out_dist_dev: *mut f32, out_count_dev: *mut u32, per_query_stats_dev: *mut u32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_hnsw_search_f64(h: *mut CozoGpuHnsw, queries: *const f64, B: u32, k: u32, ef: u32, radius: f64, row_mask: *const u32, out_ids: *mut u32, out_dist: *mut f64, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_hnsw_search_scatter_dev(h: *mut CozoGpuHnsw, queries_dev: *const f32, B: u32, k: u32, ef: u32, radius: f64, n_dest: u32, dest_ids_ptrs: *const u64, dest_dist_ptrs: *const u64, slot: u32, per_query_stats_dev: *mut u32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_hnsw_build(out: *mut *mut CozoGpuHnsw, desc: *const CozoGpuHnswBuildDesc) -> c_int;
    pub fn cozo_gpu_hnsw_insert(h: *mut CozoGpuHnsw, vectors: *const f32, count: u32, vectors_on_device: i32, ef_construction: u32, keep_pruned_connections: i32, first_id: *mut u32) -> c_int;
    pub fn cozo_gpu_hnsw_insert_at(h: *mut CozoGpuHnsw, positions: *const u32, vectors: *const f32, count: u32, vectors_on_device: i32, ef_construction: u32, keep_pruned_connections: i32, out_ids: *mut u32) -> c_int;
    pub fn cozo_gpu_hnsw_remove(h: *mut CozoGpuHnsw, ids: *const u32, count: u32) -> c_int;
    pub fn cozo_gpu_hnsw_compact(h: *mut CozoGpuHnsw, old_to_new: *mut u32) -> c_int;
    pub fn cozo_gpu_hnsw_update(h: *mut CozoGpuHnsw, ids: *const u32, vectors: *const f32, count: u32, ef_construction: u32, keep_pruned_connections: i32) -> c_int;
    pub fn cozo_gpu_hnsw_info(h: *mut CozoGpuHnsw, n_vectors: *mut u32, dim: *mut u32, n_levels: *mut u32, entry_point: *mut u32) -> c_int;
    pub fn cozo_gpu_hnsw_level_size(h: *mut CozoGpuHnsw, level: u32, n_nodes: *mut u32, n_edges: *mut u64) -> c_int;
    pub fn cozo_gpu_hnsw_export_level(h: *mut CozoGpuHnsw, level: u32, node_ids: *mut u32, row_ptr: *mut u64, col_idx: *mut u32) -> c_int;
    pub fn cozo_gpu_hnsw_export_level_dist(h: *mut CozoGpuHnsw, level: u32, dist: *mut f32) -> c_int;
    pub fn cozo_gpu_hnsw_export_live(h: *mut CozoGpuHnsw, live: *mut u8) -> c_int;
    pub fn cozo_gpu_hnsw_vectors_dev(h: *mut CozoGpuHnsw, row_stride: *mut u32) -> *const f32;
    pub fn cozo_gpu_topk_merge_dev(dist_dev: *const f32, ids_dev: *const u32, n_shards: u32, B: u32, k: u32, shard_offsets_dev: *const u64, out_ids_dev: *mut u64, out_dist_dev: *mut f32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_shards_unique_id(id: *mut u8) -> c_int;
    pub fn cozo_gpu_shards_init(out: *mut *mut CozoGpuShards, id: *const u8, rank: c_int, world: c_int) -> c_int;
    pub fn cozo_gpu_shards_free(s: *mut CozoGpuShards);
    pub fn cozo_gpu_shards_info(s: *mut CozoGpuShards, rank: *mut c_int, world: *mut c_int, exchange: *mut c_int, total_rows: *mut u64) -> c_int;
    pub fn cozo_gpu_hnsw_stage_sharded(s: *mut CozoGpuShards, local_shard: *mut CozoGpuHnsw, out_global_offset: *mut u64, out_total_rows: *mut u64) -> c_int;
    pub fn cozo_gpu_hnsw_search_sharded(s: *mut CozoGpuShards, queries: *const f32, B: u32, k: u32, ef: u32, radius: f64, root: c_int, out_ids: *mut u64, out_dist: *mut f32, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_hnsw_search_sharded_dev(s: *mut CozoGpuShards, queries_dev: *const f32, B: u32, k: u32, ef: u32, radius: f64, out_ids_dev: *mut u64, out_dist_dev: *mut f32, per_query_stats_dev: *mut u32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_hnsw_search_sharded_filtered(s: *mut CozoGpuShards, queries: *const f32, B: u32, k: u32, ef: u32, radius: f64, root: c_int, row_mask: *const u32, out_ids: *mut u64, out_dist: *mut f32, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_hnsw_search_sharded_filtered_dev(s: *mut CozoGpuShards, queries_dev: *const f32, B: u32, k: u32, ef: u32, radius: f64, row_mask_dev: *const u32, out_ids_dev: *mut u64, out_dist_dev: *mut f32, per_query_stats_dev: *mut u32, stream: *mut c_void) -> c_int;
    pub fn cozo_gpu_hnsw_search_sharded_f64(s: *mut CozoGpuShards, queries: *const f64, B: u32, k: u32, ef: u32, radius: f64, root: c_int, row_mask: *const u32, out_ids: *mut u64, out_dist: *mut f64, out_count: *mut u32, stats: *mut CozoGpuSearchStats) -> c_int;
    pub fn cozo_gpu_graph_stage(out: *mut *mut CozoGpuGraph, n: u32, m: u64, src: *const u32, dst: *const u32, w_or_null: *const f32) -> c_int;
    pub fn cozo_gpu_graph_free(g: *mut CozoGpuGraph);
    pub fn cozo_gpu_graph_stage_keys(out: *mut *mut CozoGpuGraph, m: u64, key_bytes: *const u8, key_off: *const u64, w_or_null: *const f32, undirected: i32, out_n: *mut u32) -> c_int;
    pub fn cozo_gpu_graph_node_endpoints(g: *mut CozoGpuGraph, out_first: *mut u64) -> c_int;
    pub fn cozo_gpu_graph_lookup_keys(g: *mut CozoGpuGraph, key_bytes: *const u8, key_off: *const u64, count: u32, out_ids: *mut u32) -> c_int;
    pub fn cozo_gpu_graph_export(g: *mut CozoGpuGraph, out_ptr: *mut u32, out_idx: *mut u32, out_w: *mut f32, in_ptr: *mut u32, in_idx: *mut u32) -> c_int;
    pub fn cozo_gpu_pagerank(g: *mut CozoGpuGraph, damping: f32, tol: f64, max_iter: u32, out_scores: *mut f32, out_iters: *mut u32, out_err: *mut f64, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_sssp_multi(g: *mut CozoGpuGraph, sources: *const u32, n_src: u32, out_dist: *mut f32, out_pred: *mut u32, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_sssp_goals(g: *mut CozoGpuGraph, sources: *const u32, n_src: u32, goals: *const u32, n_goals: u32, keep_ties: i32, out_cost: *mut f32, out_path_off: *mut u64, out_paths: *mut u32, paths_cap: u64, out_tie_off: *mut u64, out_tie_edges: *mut u32, ties_cap: u64, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_sssp_paths(g: *mut CozoGpuGraph, sources: *const u32, goals: *const u32, n_src: u32, forb_node_ptr: *const u32, forb_nodes: *const u32, forb_edge_ptr: *const u32, forb_edge_src: *const u32, forb_edge_dst: *const u32, max_len: u32, out_cost: *mut f32, out_len: *mut u32, out_paths: *mut u32, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_closeness(g: *mut CozoGpuGraph, out: *mut f32, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_betweenness(g: *mut CozoGpuGraph, out: *mut f32, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
    pub fn cozo_gpu_clustering(g: *mut CozoGpuGraph, out_cc: *mut f64, out_triangles: *mut u64, out_degree: *mut u64, out_kernel_ms: *mut f64, poison: *const c_int) -> c_int;
}
