//! hnsw_gpu.rs — staging of an HNSW index relation onto the device and the batched k-NN operator.
//!
//! Destination: cozo-core/src/runtime/hnsw_gpu.rs under `#[cfg(feature = "gpu-b200")]`.
//! Not compiled in the build image (no Rust toolchain).  The executable twin is
//! cozo_b200/host/hnsw.hpp (`StagedHnswIndex::stage`, `hnsw_knn_batch`, `HnswSearchRA::iter`),
//! which the GPU tests drive against the oracle.
//!
//! Three pieces:
//!   1. `StagedIndex::stage`   — one scan of `rel:idx` + point reads of the base relation
//!                               → CozoGpuHnswStageDesc → cozo_gpu_hnsw_stage.
//!   2. `SessionTx::hnsw_knn_batch` — the body of `hnsw_knn` (runtime/hnsw.rs:869-1012) for B
//!                               query vectors at once: ONE cozo_gpu_hnsw_search, then the
//!                               reference's own per-candidate tuple assembly, bindings and filter.
//!   3. `HnswSearchRA::iter_gpu` — `HnswSearchRA::iter` (query/ra.rs:1085-1121) restated to collect
//!                               parent tuples into batches instead of calling hnsw_knn per tuple.

use std::collections::BTreeMap;
use std::ptr;
use std::sync::{Arc, Mutex};

use itertools::Itertools;
use miette::{bail, miette, Result};

use crate::data::expr::{eval_bytecode_pred, Bytecode};
use crate::data::tuple::Tuple;
use crate::data::value::{DataValue, Vector};
use crate::gpu::sys::*;
use crate::parse::sys::VecElementType;
use crate::parse::SourceSpan;
use crate::runtime::hnsw::{CompoundKey, HnswIndexManifest};
use crate::runtime::relation::RelationHandle;
use crate::runtime::transact::SessionTx;
use crate::query::ra::HnswSearchRA; // for iter_gpu below
use crate::parse::sys::HnswSearch;

fn check(rc: std::os::raw::c_int) -> Result<()> {
    if rc == COZO_GPU_OK {
        return Ok(());
    }
    let msg = unsafe { std::ffi::CStr::from_ptr(cozo_gpu_last_error()) };
    Err(miette!("gpu-b200: {}", msg.to_string_lossy()))
}

/// Device-resident cache of one `rel:idx` relation.  Dense id = rank of the compound key
/// `(tuple_key, field_idx, sub_idx)` among the layer-0 self-loop rows, i.e. key order.
pub(crate) struct StagedIndex {
    h: *mut CozoGpuHnsw,
    keys: Vec<CompoundKey>,
    /// (base relation id, index relation id) the copy was staged from.
    stamp: (u64, u64),
    /// manifest.dtype == F64: distances in f64 through cozo_gpu_hnsw_search_f64
    f64_index: bool,
}

/// The reference keeps no index version counter, so the device copy is dropped AT the mutation sites
/// (one added line each, INTEGRATION.md §2 lists them):
///   hnsw_put    <- query/stored.rs:332, :630 and runtime/relation.rs:1177 (create_hnsw_index bulk insert)
///   hnsw_remove <- query/stored.rs:995-997
///   index drop  <- runtime/relation.rs:1383 (`hnsw_indices.remove`)
/// each calls `gpu_index_invalidate(idx_handle.id)` before touching the relation, except that a `:put` whose
/// compound keys are all new goes through `gpu_index_put_new_keys`, and `:rm` through `gpu_index_remove_keys`,
/// instead.  The next search re-stages a dropped copy (changed vectors can likewise go to cozo_gpu_hnsw_update —
/// `StagedHnswIndex::put_rows` in the C++ twin shows the exact rules).
/// A staged copy is only handed to readers whose transaction started after the staging.
pub(crate) fn gpu_index_invalidate(idx_rel_id: crate::runtime::relation::RelationId) {
    STAGED.lock().unwrap().remove(&idx_rel_id.0);
}

/// hnsw_put of compound keys the staged copy does not hold yet, at any key position (query/stored.rs:332 ->
/// hnsw.rs:679-727), absorbed in place by cozo_gpu_hnsw_insert_at.  `new`: (key, vector) in key order.  The device
/// moves every existing id up by the number of new keys before it, so `keys` stays the key order the entry-point
/// rule reads.  F64 copies (search-only on the device) and copies still shared with a reader are dropped instead:
/// the next search re-stages them.
pub(crate) fn gpu_index_put_new_keys(
    idx_rel_id: crate::runtime::relation::RelationId,
    new: &[(CompoundKey, Vec<f32>)],
    mf: &HnswIndexManifest,
) -> Result<()> {
    let mut map = STAGED.lock().unwrap();
    let Some(arc) = map.get_mut(&idx_rel_id.0) else { return Ok(()) };
    let staged = match Arc::get_mut(arc) {
        Some(s) if !s.f64_index => s,
        _ => {
            map.remove(&idx_rel_id.0);
            return Ok(());
        }
    };
    // lower_bound in the id -> key table; removed ids keep their ids (and keys) until a re-stage
    let positions: Vec<u32> = new.iter().map(|(k, _)| staged.keys.partition_point(|x| x < k) as u32).collect();
    let flat: Vec<f32> = new.iter().flat_map(|(_, v)| v.iter().copied()).collect();
    let mut ids = vec![0u32; new.len()];
    let rc = unsafe {
        cozo_gpu_hnsw_insert_at(staged.h, positions.as_ptr(), flat.as_ptr(), new.len() as u32, 0,
                                mf.ef_construction as u32, mf.keep_pruned_connections as i32, ids.as_mut_ptr())
    };
    if let Err(e) = check(rc) {
        map.remove(&idx_rel_id.0); // the copy may be half updated: re-stage on the next search
        return Err(e);
    }
    for (i, (k, _)) in new.iter().enumerate() {
        staged.keys.insert(ids[i] as usize, k.clone()); // ids ascend: key i lands after keys 0..i
    }
    Ok(())
}

/// hnsw_remove of whole tuples (query/stored.rs:995-997 -> hnsw.rs:728-753), absorbed in place: every compound key
/// of each removed tuple key goes to cozo_gpu_hnsw_remove, then cozo_gpu_hnsw_compact drops the removed ids, so the
/// copy stays in the id space a fresh staging of the relation gives (dense id = key rank of the remaining rows).
/// F64 copies, copies still shared with a reader, and any error drop the copy instead: the next search re-stages it.
pub(crate) fn gpu_index_remove_keys(idx_rel_id: crate::runtime::relation::RelationId, tuple_keys: &[Tuple]) -> Result<()> {
    let mut map = STAGED.lock().unwrap();
    let Some(arc) = map.get_mut(&idx_rel_id.0) else { return Ok(()) };
    let staged = match Arc::get_mut(arc) {
        Some(s) if !s.f64_index => s,
        _ => {
            map.remove(&idx_rel_id.0);
            return Ok(());
        }
    };
    // the compound keys (key, field, sub_idx) of one tuple key are consecutive in the id -> key table
    let mut ids: Vec<u32> = Vec::new();
    for tk in tuple_keys {
        let lo = staged.keys.partition_point(|x| x.0 < *tk);
        ids.extend((lo..staged.keys.len()).take_while(|&i| staged.keys[i].0 == *tk).map(|i| i as u32));
    }
    if ids.is_empty() {
        return Ok(());
    }
    let mut old_to_new = vec![0u32; staged.keys.len()];
    let rc = unsafe { cozo_gpu_hnsw_remove(staged.h, ids.as_ptr(), ids.len() as u32) };
    let rc = if rc == COZO_GPU_OK { unsafe { cozo_gpu_hnsw_compact(staged.h, old_to_new.as_mut_ptr()) } } else { rc };
    if let Err(e) = check(rc) {
        map.remove(&idx_rel_id.0); // the copy may be half updated: re-stage on the next search
        return Err(e);
    }
    let mut id = 0usize;
    staged.keys.retain(|_| {
        id += 1;
        old_to_new[id - 1] != COZO_GPU_NONE
    });
    Ok(())
}

unsafe impl Send for StagedIndex {}
unsafe impl Sync for StagedIndex {}

impl Drop for StagedIndex {
    fn drop(&mut self) {
        unsafe { cozo_gpu_hnsw_free(self.h) }
    }
}

lazy_static::lazy_static! {
    /// (idx relation id) -> staged copy; lives as long as the Db.
    static ref STAGED: Mutex<BTreeMap<u64, Arc<StagedIndex>>> = Mutex::new(BTreeMap::new());
}

impl StagedIndex {
    pub(crate) fn get_or_stage(
        tx: &SessionTx<'_>,
        base: &RelationHandle,
        idx: &RelationHandle,
        mf: &HnswIndexManifest,
    ) -> Result<Arc<StagedIndex>> {
        crate::fixed_rule::algos::gpu::ensure_device()?; // no CPU fallback: surfaces the init error
        let stamp = (base.id.0, idx.id.0);
        let mut map = STAGED.lock().unwrap();
        if let Some(s) = map.get(&idx.id.0) {
            if s.stamp == stamp {
                return Ok(s.clone());
            }
        }
        let s = Arc::new(Self::stage(tx, base, idx, mf, stamp)?);
        map.insert(idx.id.0, s.clone());
        Ok(s)
    }

    fn stage(
        tx: &SessionTx<'_>,
        base: &RelationHandle,
        idx: &RelationHandle,
        mf: &HnswIndexManifest,
        stamp: (u64, u64),
    ) -> Result<Self> {
        let f64_index = mf.dtype == VecElementType::F64; // f64 payloads, searched by cozo_gpu_hnsw_search_f64
        let k = base.metadata.keys.len();
        // index rows: (layer, fr_k.., fr__field, fr__sub_idx, to_k.., to__field, to__sub_idx,
        //              dist, hash, ignore_link)   — runtime/relation.rs:1064-1126
        let fr_key = |t: &Tuple| -> Option<CompoundKey> {
            let fld = t[k + 1].get_int()?; // Null on the canary row (hnsw.rs:903-909)
            Some((t[1..k + 1].to_vec(), fld as usize, t[k + 2].get_int().unwrap() as i32))
        };
        let to_key = |t: &Tuple| -> CompoundKey {
            (
                t[k + 3..2 * k + 3].to_vec(),
                t[2 * k + 3].get_int().unwrap() as usize,
                t[2 * k + 4].get_int().unwrap() as i32,
            )
        };
        // pass 1 (layer 0 only): the dictionary.  scan_all is in key order, layers are <= 0, so the
        // layer-0 rows are the LAST block; self-loop rows name every indexed vector.
        let rows: Vec<Tuple> = idx.scan_all(tx).try_collect()?;
        let mut ids: BTreeMap<CompoundKey, u32> = BTreeMap::new();
        for t in rows.iter().filter(|t| t[0].get_int() == Some(0)) {
            if let Some(f) = fr_key(t) {
                ids.entry(f).or_insert(0);
            }
        }
        let keys: Vec<CompoundKey> = ids.keys().cloned().collect();
        for (i, v) in ids.values_mut().enumerate() {
            *v = i as u32;
        }
        let n = keys.len();
        // entry point = first row with layer in [i64::MIN, 1] (hnsw.rs:891-899)
        let (entry, bottom_level) = match rows.first().and_then(|t| fr_key(t).map(|f| (f, t[0].get_int().unwrap()))) {
            Some((f, l)) => (*ids.get(&f).ok_or_else(|| miette!("corrupted index"))?, l),
            None => (COZO_GPU_NONE, 0),
        };
        let n_levels = if entry == COZO_GPU_NONE { 1 } else { (-bottom_level) as usize + 1 };
        // pass 2: adjacency under the reading rules of hnsw_get_neighbours(include_deleted = false)
        // (hnsw.rs:586-626): drop rows whose `to` TUPLE key equals the `fr` tuple key, drop
        // ignore_link rows; neighbours stay in key order.
        let mut adj: Vec<BTreeMap<u32, Vec<u32>>> = vec![BTreeMap::new(); n_levels];
        for t in &rows {
            let layer = t[0].get_int().unwrap();
            if layer > 0 {
                continue;
            }
            let f = match fr_key(t) {
                Some(f) => f,
                None => continue,
            };
            let l = (-layer) as usize;
            let row = adj[l].entry(ids[&f]).or_default();
            let to = to_key(t);
            if to.0 == f.0 || t[2 * k + 7].get_bool() == Some(true) {
                continue;
            }
            row.push(*ids.get(&to).ok_or_else(|| miette!("corrupted index"))?);
        }
        // vectors: VectorCache::ensure_key (hnsw.rs:122-151)
        let mut vectors = vec![0f32; if f64_index { 0 } else { n * mf.vec_dim }];
        let mut vectors64 = vec![0f64; if f64_index { n * mf.vec_dim } else { 0 }];
        for (i, key) in keys.iter().enumerate() {
            let row = base.get(tx, &key.0)?.ok_or_else(|| miette!("Cannot find compound key for HNSW"))?;
            let field = if key.2 >= 0 {
                match &row[key.1] {
                    DataValue::List(l) => &l[key.2 as usize],
                    d => bail!("Cannot interpret {} as list", d),
                }
            } else {
                &row[key.1]
            };
            match field {
                DataValue::Vec(Vector::F32(v)) if v.len() == mf.vec_dim && !f64_index => {
                    vectors[i * mf.vec_dim..(i + 1) * mf.vec_dim].copy_from_slice(v.as_slice().unwrap())
                }
                DataValue::Vec(Vector::F64(v)) if v.len() == mf.vec_dim && f64_index => {
                    vectors64[i * mf.vec_dim..(i + 1) * mf.vec_dim].copy_from_slice(v.as_slice().unwrap())
                }
                d => bail!("Cannot interpret {} as vector", d),
            }
        }
        // flatten
        let mut node_ids: Vec<Vec<u32>> = vec![vec![]; n_levels];
        let mut row_ptr: Vec<Vec<u64>> = vec![vec![0]; n_levels];
        let mut col_idx: Vec<Vec<u32>> = vec![vec![]; n_levels];
        for l in 0..n_levels {
            if l == 0 {
                for i in 0..n as u32 {
                    if let Some(r) = adj[0].get(&i) {
                        col_idx[0].extend_from_slice(r);
                    }
                    row_ptr[0].push(col_idx[0].len() as u64);
                }
            } else {
                for (i, r) in &adj[l] {
                    node_ids[l].push(*i);
                    col_idx[l].extend_from_slice(r);
                    row_ptr[l].push(col_idx[l].len() as u64);
                }
            }
        }
        let levels: Vec<CozoGpuHnswLevel> = (0..n_levels)
            .map(|l| CozoGpuHnswLevel {
                n_nodes: if l == 0 { n as u32 } else { node_ids[l].len() as u32 },
                node_ids: if l == 0 { ptr::null() } else { node_ids[l].as_ptr() },
                row_ptr: row_ptr[l].as_ptr(),
                col_idx: col_idx[l].as_ptr(),
            })
            .collect();
        let desc = CozoGpuHnswStageDesc {
            n_vectors: n as u32,
            dim: mf.vec_dim as u32,
            metric: metric_code(mf.distance),
            n_levels: n_levels as u32,
            levels: levels.as_ptr(),
            vectors: if f64_index { vectors64.as_ptr() as *const _ } else { vectors.as_ptr() as *const _ },
            vectors_on_device: 0,
            entry_point: entry,
            m_max0: mf.m_max0 as u32,
            m_max: mf.m_max as u32,
            vec_dtype: f64_index as i32,
        };
        let mut h = ptr::null_mut();
        check(unsafe { cozo_gpu_hnsw_stage(&mut h, &desc) })?;
        Ok(StagedIndex { h, keys, stamp, f64_index })
    }
}

impl<'a> SessionTx<'a> {
    /// `hnsw_knn` (runtime/hnsw.rs:869-1012) for a batch of query vectors.  Returns, per query,
    /// exactly the tuples `hnsw_knn` returns, in the same order.
    pub(crate) fn hnsw_knn_batch(
        &self,
        qs: &[Vector],
        config: &HnswSearch,
        filter_bytecode: &Option<(Vec<Bytecode>, SourceSpan)>,
        stack: &mut Vec<DataValue>,
    ) -> Result<Vec<Vec<Tuple>>> {
        let dim = config.manifest.vec_dim;
        let staged = StagedIndex::get_or_stage(self, &config.base_handle, &config.idx_handle, &config.manifest)?;
        // the query is cast to the index dtype (hnsw.rs:879-884)
        let mut flat = Vec::with_capacity(if staged.f64_index { 0 } else { qs.len() * dim });
        let mut flat64 = Vec::with_capacity(if staged.f64_index { qs.len() * dim } else { 0 });
        for q in qs {
            if q.len() != dim {
                bail!("query vector dimension mismatch"); // hnsw.rs:876-878
            }
            match (q, staged.f64_index) {
                (Vector::F32(v), false) => flat.extend(v.iter().copied()),
                (Vector::F64(v), false) => flat.extend(v.iter().map(|x| *x as f32)), // hnsw.rs:883
                (Vector::F32(v), true) => flat64.extend(v.iter().map(|x| *x as f64)), // hnsw.rs:882
                (Vector::F64(v), true) => flat64.extend(v.iter().copied()),
            }
        }
        // With a filter the reference keeps all ef results and filters before truncating to k
        // (hnsw.rs:942-946, 1001-1008).  If the bytecode never reads the bound distance, its verdict is a
        // property of the indexed row: evaluate it once per row, ship the verdicts as a bit mask and let the
        // kernel trim to k after filtering (cozo_gpu_hnsw_search_filtered).  Otherwise ask for all ef
        // candidates and filter here.
        let nk = config.base_handle.metadata.keys.len();
        let dist_pos = self.distance_binding_pos(config);
        let device_filter = match (filter_bytecode, dist_pos) {
            (Some((code, _)), Some(p)) => !code.iter().any(|bc| matches!(bc, Bytecode::Binding { tuple_pos: Some(tp), .. } if *tp == p)),
            (Some(_), None) => true,
            (None, _) => false,
        };
        let k_dev = if filter_bytecode.is_some() && !device_filter { config.ef } else { config.k.min(config.ef) };
        let b = qs.len();
        let mut ids = vec![COZO_GPU_NONE; b * k_dev];
        let mut dist = vec![0f32; b * k_dev];
        let mut dist64 = vec![0f64; if staged.f64_index { b * k_dev } else { 0 }];
        let mut count = vec![0u32; b];
        let mut stats = CozoGpuSearchStats::default();
        let mut mask = vec![];
        if device_filter {
            let (code, span) = filter_bytecode.as_ref().unwrap();
            mask = vec![0u32; (staged.keys.len() + 31) / 32 + 1];
            for (id, key) in staged.keys.iter().enumerate() {
                let cand = self.assemble_candidate(config, key, nk, DataValue::Null)?; // distance slot unused by the filter
                if eval_bytecode_pred(code, &cand, stack, *span)? {
                    mask[id >> 5] |= 1 << (id & 31);
                }
            }
        }
        if staged.f64_index {
            check(unsafe {
                cozo_gpu_hnsw_search_f64(
                    staged.h, flat64.as_ptr(), b as u32, k_dev as u32, config.ef as u32, config.radius.unwrap_or(-1.0),
                    if device_filter { mask.as_ptr() } else { ptr::null() },
                    ids.as_mut_ptr(), dist64.as_mut_ptr(), count.as_mut_ptr(), &mut stats,
                )
            })?;
        } else if device_filter {
            check(unsafe {
                cozo_gpu_hnsw_search_filtered(
                    staged.h, flat.as_ptr(), b as u32, k_dev as u32, config.ef as u32, config.radius.unwrap_or(-1.0),
                    mask.as_ptr(), ids.as_mut_ptr(), dist.as_mut_ptr(), count.as_mut_ptr(), &mut stats,
                )
            })?;
        } else {
            check(unsafe {
                cozo_gpu_hnsw_search(
                    staged.h, flat.as_ptr(), b as u32, k_dev as u32, config.ef as u32,
                    config.radius.unwrap_or(-1.0), // < 0: no radius
                    ids.as_mut_ptr(), dist.as_mut_ptr(), count.as_mut_ptr(), &mut stats,
                )
            })?;
        }
        let mut out = Vec::with_capacity(b);
        for qi in 0..b {
            let mut ret = vec![];
            for j in 0..count[qi] as usize {
                let cand_key = &staged.keys[ids[qi * k_dev + j] as usize];
                let distance = if staged.f64_index { dist64[qi * k_dev + j] } else { dist[qi * k_dev + j] as f64 };
                let cand_tuple = self.assemble_candidate(config, cand_key, nk, DataValue::from(distance))?;
                if let (Some((code, span)), false) = (filter_bytecode, device_filter) {
                    if !eval_bytecode_pred(code, &cand_tuple, stack, *span)? {
                        continue;
                    }
                }
                ret.push(cand_tuple);
            }
            ret.truncate(config.k); // device results are already nearest-first (hnsw.rs:1005-1006)
            out.push(ret);
        }
        Ok(out)
    }
}

impl<'a> SessionTx<'a> {
    /// base row ++ bindings in the order of `HnswSearch::all_bindings` (hnsw.rs:958-995, program.rs:1016-1025)
    fn assemble_candidate(&self, config: &HnswSearch, cand_key: &CompoundKey, nk: usize, distance: DataValue) -> Result<Tuple> {
        let mut cand_tuple = config.base_handle.get(self, &cand_key.0)?.ok_or_else(|| miette!("corrupted index"))?;
        if config.bind_field.is_some() {
            let field = if cand_key.1 < nk {
                config.base_handle.metadata.keys[cand_key.1].name.clone()
            } else {
                config.base_handle.metadata.non_keys[cand_key.1 - nk].name.clone()
            };
            cand_tuple.push(DataValue::Str(field));
        }
        if config.bind_field_idx.is_some() {
            cand_tuple.push(if cand_key.2 < 0 { DataValue::Null } else { DataValue::from(cand_key.2 as i64) });
        }
        if config.bind_distance.is_some() {
            cand_tuple.push(distance);
        }
        if config.bind_vector.is_some() {
            let vec = if cand_key.2 < 0 {
                cand_tuple[cand_key.1].clone()
            } else {
                match &cand_tuple[cand_key.1] {
                    DataValue::List(v) => v[cand_key.2 as usize].clone(),
                    v => bail!("corrupted index value {:?}", v),
                }
            };
            cand_tuple.push(vec);
        }
        Ok(cand_tuple)
    }
    /// position of the bound distance inside the candidate tuple, if it is bound at all
    fn distance_binding_pos(&self, config: &HnswSearch) -> Option<usize> {
        config.bind_distance.as_ref()?;
        let arity = config.base_handle.metadata.keys.len() + config.base_handle.metadata.non_keys.len();
        Some(arity + config.bind_field.is_some() as usize + config.bind_field_idx.is_some() as usize)
    }
}

/// Parent tuples gathered per device call.  One launch amortises best from a few hundred queries
/// up; smaller parents simply produce one short batch.
const GPU_BATCH: usize = 4096;

impl HnswSearchRA {
    /// `HnswSearchRA::iter` (query/ra.rs:1085-1121), batching the parent's tuples.
    pub(crate) fn iter_gpu<'a>(
        &'a self,
        tx: &'a SessionTx<'_>,
        delta_rule: Option<&crate::data::program::MagicSymbol>,
        stores: &'a BTreeMap<crate::data::program::MagicSymbol, crate::runtime::temp_store::EpochStore>,
    ) -> Result<crate::query::ra::TupleIter<'a>> {
        let bindings = self.parent.bindings_after_eliminate();
        let bind_idx = bindings
            .iter()
            .position(|b| *b == self.hnsw_search.query)
            .unwrap_or(usize::MAX);
        let config = self.hnsw_search.clone();
        let filter_code = self.filter_bytecode.clone();
        let mut stack = vec![];
        let chunks = self.parent.iter(tx, delta_rule, stores)?.chunks(GPU_BATCH);
        let mut out: Vec<Result<Tuple>> = vec![];
        for chunk in &chunks {
            let tuples: Vec<Tuple> = chunk.try_collect()?;
            let mut qs = Vec::with_capacity(tuples.len());
            for t in &tuples {
                match &t[bind_idx] {
                    DataValue::Vec(v) => qs.push(v.clone()),
                    d => bail!("Expected vector, got {:?}", d),
                }
            }
            let res = tx.hnsw_knn_batch(&qs, &config, &filter_code, &mut stack)?;
            for (tuple, rows) in tuples.into_iter().zip(res) {
                for r in rows {
                    let mut o = tuple.clone();
                    o.extend(r);
                    out.push(Ok(o));
                }
            }
        }
        Ok(Box::new(out.into_iter()))
    }
}

/// HnswDistance (parse/sys.rs:94-98) is declared `L2, InnerProduct, Cosine`; the C ABI numbers
/// them COZO_GPU_L2 = 0, COZO_GPU_COSINE = 1, COZO_GPU_IP = 2.
pub(crate) fn metric_code(d: crate::parse::sys::HnswDistance) -> i32 {
    use crate::parse::sys::HnswDistance::*;
    match d {
        L2 => COZO_GPU_L2,
        Cosine => COZO_GPU_COSINE,
        InnerProduct => COZO_GPU_IP,
    }
}
